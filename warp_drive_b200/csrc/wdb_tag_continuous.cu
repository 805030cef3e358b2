// wdb_tag_continuous.cu -- TagContinuous env.step() and the fused rollout step for sm_90a.
//
// Replaces CudaTagContinuousStep + CudaTagContinuousGenerateObservation +
// CudaTagContinuousComputeReward (example_envs/tag_continuous/
// tag_continuous_step_pycuda.cu:13-520 of the reference) and -- in the fused entry point
// wdb_tag_continuous_rollout_step -- also sample_actions x2 (core/random.cu:51-85), the
// action/reward/done push-to-batch copies and episodic bookkeeping of the trainer
// (trainer_base.py:437-601) and the 13 reset launches (core/reset.cu:9-75,
// pycuda_function_manager.py:668-753) of one rollout timestep.
//
// Layout / mapping
//   * one thread per agent; a CTA carries EPB whole env replicas (EPB*N threads) so warps
//     stay full when N is not a multiple of 32 (N=105 -> 3 envs = 315 threads = 10 warps,
//     98.4 % of lanes busy; the reference's 105-thread block wastes 18 % of its 4th warp).
//   * agent state (x, y, speed, acc, dir, alive) is loaded once with unit-stride loads,
//     updated in registers, written back once, and staged in shared memory; the O(N^2)
//     neighbour sweep and the tagger scan read only shared memory.  The reference re-reads
//     global memory per pair and keeps N*(N-1) distances and ids per env in global scratch.
//   * action probabilities arrive in shared memory by TMA bulk copies (cp.async.bulk +
//     mbarrier) issued first thing (the reference reads rows with an A*4-byte stride per
//     thread and round-trips the CDF through global memory); observations are assembled in
//     a shared-memory tile laid out like their destination and leave by TMA bulk stores
//     that overlap the reward phase.
//   * every global read of the prologue is issued back to back before the first global
//     store (one memory round trip).
//
// Exactness (what "parity" means here; tests/test_gpu_envs.py compares against the
// reference kernels compiled from the reference sources, bit for bit)
//   * kinematics use the same float32 expressions as the reference.
//   * k-nearest selection: the reference orders neighbours by
//     d = (float)sqrt(pow((double)dx,2)+pow((double)dy,2)) through a swap-based partial
//     selection sort whose tie order is NOT id order (:179-199).  The fast paths -- a
//     temporal-coherence threshold scan on packed float32x2 arithmetic that keeps a bit
//     mask of the ~K+2 candidates inside last step's neighbour radius, or a branch-free
//     sorting network over all candidates -- rank packed (float32 squared distance | id)
//     keys and accept the result only when the exact float32 squared distances of the
//     K+1 nearest are strictly increasing with relative gaps > 2^-19 (2^-15 for the last
//     pair, which also covers the key truncation) -- then the ranking provably equals the
//     ranking by d and no tie exists.  Otherwise the agent takes the exact path: the
//     literal reference algorithm on float64-derived distances.
//   * dx / (sqrt(2.0)*L) is a float64 division in the reference; here it is a float64
//     multiply by the reciprocal plus a check that the product is not within 4 ulp of a
//     float32 rounding boundary (else the true division runs), which gives the same bits.
//   * tag test: a float32 pre-test with a guard band decides "clearly not tagged"; anything
//     near the margin re-evaluates with the reference's float64 expression.
//   * the reference's two data races (rewards[tagger] += ..., num_runners -= 1, :324-329)
//     are resolved with shared-memory atomics (every tag counts), matching the reference's
//     NumPy semantics (tag_continuous.py:660-672).
#include "wdb_tc_common.cuh"

namespace {

// ACTS_IN (fused only): the policy forward already sampled this step's actions into
// Q.actions_batch (wdb_mlp_policy_forward_sampled); they are read instead of sampled, so no
// probability tile, no TMA and no RNG.
template <bool FUSED, int MAXT, bool ACTS_IN = false>
__global__ void __launch_bounds__(MAXT, MAXT == 320 ? 2 : 1)
tag_continuous_kernel(const __grid_constant__ TcParams P, const __grid_constant__ FusedParams Q) {
  static_assert(FUSED || !ACTS_IN, "actions in the batch is a mode of the fused step");
  extern __shared__ __align__(16) unsigned char smem_raw[];
#ifdef WDB_PHASE_CLOCKS
  const long long wdb_t0 = clock64();
#endif
  const int N = P.N, epb = P.epb, K = P.K;
  const int EN = epb * N;
  const int nwarps = blockDim.x / kWarp;
  // selection keys: x / y of every agent as separate planes (dead agents and the padding up
  // to a multiple of 16 = +inf), 16-byte aligned rows so the scan reads 4 candidates per load
  const int Ne = tc_key_stride(N);
  float *skx = reinterpret_cast<float *>(smem_raw);
  float *sky = skx + epb * Ne;
  float2 *spos = reinterpret_cast<float2 *>(sky + epb * Ne);   // real positions
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
  int *s_rowbase = s_ntag + 4;    // [N] offset of the agent's obs row inside the tile
  int *s_rowstride = s_rowbase + N;  // [N] tile stride between consecutive envs
  unsigned long long *s_mbar = reinterpret_cast<unsigned long long *>(
      smem_raw + tc_small_bytes(epb, N) - 16);   // 8-byte aligned mbarrier
  // per-warp scratch (history candidate list, then the exact path's distance/id lists)
  unsigned char *s_scr = smem_raw + tc_small_bytes(epb, N);
  // big tile: action probabilities first (fused mode), then the observation tile
  float *s_tile = reinterpret_cast<float *>(s_scr + (size_t)nwarps * P.scr_warp_bytes);

  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const int le = tid / N;
  const int a = tid - le * N;
  // CTAs past full_ctas carry ONE env each (see plan_packed: the last, partly filled wave)
  const bool tail_cta = (int)blockIdx.x >= P.full_ctas;
  const int env0 = P.env_begin + (tail_cta ? P.full_ctas * epb + ((int)blockIdx.x - P.full_ctas)
                                           : (int)blockIdx.x * epb);
  const int env = env0 + le;
  const int envs_here = tail_cta ? min(1, P.env_end - env0) : min(epb, P.env_end - env0);
  const bool active = le < envs_here;
  const int gi = env * N + a;
  const int li = le * N + a;
  const float L = P.grid_length;

  const int F = P.use_full_obs ? 7 * (N - 1) + 1 : 7 * K + 1;
  // observation tile layout == the layout of the destination the next forward pass reads:
  // per policy p a dense [epb, Np, F] block (one policy covering every agent in step-only
  // mode), so the copy-out is a plain contiguous block copy per policy
  // (recomputed where it is used: four values held across the neighbour search spill)
  auto tile_base = [&](int p) {
    int acc = 0;
#pragma unroll
    for (int q = 0; q < kMaxPolicies; q++)
      if (FUSED && q < p && q < Q.n_policies) acc += F * epb * Q.policy_size[q];
    return acc;
  };

  // which blocks of the observation tile can leave through the TMA (16-byte aligned shared /
  // global addresses and size); decided here, used after the tile is complete
  uint32_t out_mask = 0;   // bit p: policy block p goes by TMA;  bit 8: the [E,N,F] array
  if (!P.use_full_obs && P.stage_obs) {
    if (!FUSED) {
      if (tma_ok(P.obs + (long long)env0 * N * F, smem_u32(s_tile), 4ull * envs_here * N * F))
        out_mask |= 1u << 8;
    } else {
#pragma unroll
      for (int p = 0; p < kMaxPolicies; p++) {
        if (p < Q.n_policies && Q.obs_next[p]) {
          const int np = Q.policy_size[p];
          if (tma_ok(Q.obs_next[p] + (long long)env0 * np * F, smem_u32(s_tile + tile_base(p)),
                     4ull * envs_here * np * F))
            out_mask |= 1u << p;
        }
      }
    }
  }

  // ---- categorical sampling of both action heads (core/random.cu:51-85): the probability
  // blocks are requested first thing (TMA), they land while the state loads fly ----
  // Block (p, head) = the [envs_here, Np, A] probabilities of this CTA's envs, contiguous in
  // global memory but in general NOT 16-byte aligned (taggers: 1260 bytes at a 1260 c byte
  // offset).  The TMA therefore fetches the 16-byte-aligned SUPERSET of each block (up to 15
  // bytes of neighbouring rows of the same tensor on either side) into a 16-byte-aligned
  // slot, and the rows are addressed `lead` bytes into the slot.  Slots are padded so that
  // supersets never overlap.  A block falls back to per-thread global reads only when the
  // superset would leave the tensor (unaligned tensor base / end).
  // The geometry of block q = 2 p + h is recomputed where it is needed: held in registers
  // from here to the sampling phase it would spill.
  struct ProbBlock { uint32_t lead, slot, span; bool tma; };
  auto prob_block = [&](int q) {
    ProbBlock b = {0u, 0u, 0u, false};
#pragma unroll
    for (int r = 0; r < 2 * kMaxPolicies; r++) {
      if (r > q) break;
      const int p = r >> 1, h = r & 1;
      const int np = (p < Q.n_policies) ? Q.policy_size[p] : 0;
      const int A = h ? Q.A1 : Q.A0;
      if (r < q) {
        b.slot += ((4u * epb * np * A + 15u) & ~15u) + 32u;   // room for lead + tail padding
        continue;
      }
      const float *base = (p < Q.n_policies) ? (h ? Q.probs1[p] : Q.probs0[p]) : nullptr;
      const uint32_t bytes = 4u * envs_here * np * A;
      const unsigned long long tensor_bytes = 4ull * P.n_envs * np * A;
      const uintptr_t ga = reinterpret_cast<uintptr_t>(base) + 4ull * env0 * np * A;
      b.lead = (uint32_t)(ga & 15);
      b.span = (b.lead + bytes + 15u) & ~15u;
      // with a 16-byte-aligned tensor base the superset starts inside the tensor; it must
      // also end inside it
      const bool inside = ((reinterpret_cast<uintptr_t>(base) & 15) == 0) &&
                          (4ull * env0 * np * A - b.lead + b.span <= tensor_bytes);
      b.tma = np > 0 && bytes > 0 && inside;
    }
    return b;
  };
  uint32_t tma_mask = 0;   // bit 2p / 2p+1: block (p, head) travels by TMA
  const uint32_t mbar = smem_u32(s_mbar);
  if (FUSED && !ACTS_IN) {
#pragma unroll
    for (int q = 0; q < 2 * kMaxPolicies; q++)
      if (prob_block(q).tma) tma_mask |= 1u << q;
    if (tid == 0) mbar_init(mbar, 1);      // (includes the init fence; waiters sync below)
  }

  // ------------------------------------------------------------------ phase 0
  // Every global read of the prologue is issued here, back to back, BEFORE any global store
  // (a store would pin the later loads behind it): one memory round trip instead of six.
  int g_type = 0, g_pol = 0, g_slot = 0;           // per agent id (tid < N)
  if (tid < N) {
    g_type = P.agent_types[tid];
    if (FUSED) { g_pol = Q.agent_policy[tid]; g_slot = Q.agent_slot[tid]; }
  }
  int my_pol = 0, my_slot = 0;                     // of this thread's agent
  if (FUSED && active) { my_pol = Q.agent_policy[a]; my_slot = Q.agent_slot[a]; }
  // last step's neighbour ids (history path), consumed after the kinematics
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
  if (FUSED && !ACTS_IN && active) {
    if (Q.uniforms) {
      u0 = Q.uniforms[2ll * gi];
      u1 = Q.uniforms[2ll * gi + 1];
    } else {
      rng_seed = reinterpret_cast<const RngHeader *>(Q.rng)->seed;
      rng_off = rng_offsets(Q.rng)[gi];
    }
  }
  // action -> acceleration / turn tables, staged at the head of the per-warp scratch (free
  // until the neighbour search) so that the kinematics do not wait on a dependent global load
  float *s_tab = reinterpret_cast<float *>(s_scr);
  const bool tab_ok = FUSED && (size_t)(Q.A0 + Q.A1) * 4 <= (size_t)nwarps * P.scr_warp_bytes;
  float g_tab = 0.f;
  if (tab_ok && tid < Q.A0 + Q.A1)
    g_tab = tid < Q.A0 ? P.acc_actions[tid] : P.turn_actions[tid - Q.A0];

  int act0 = 0, act1 = 0;
  if (FUSED) {
    // Programmatic dependent launch (option "pdl"): this grid may have started while the policy
    // forward was still running.  Everything above read only what the PREVIOUS env step wrote
    // (complete: the forward released us after its own griddepcontrol.wait); the probabilities
    // (or the actions the forward sampled) are requested only now.  A no-op when launched
    // without the attribute.
    griddep_wait();
    if (ACTS_IN && active) {
#pragma unroll
      for (int p = 0; p < kMaxPolicies; p++) {
        if (p == my_pol) {
          const int2 v = *reinterpret_cast<const int2 *>(
              Q.actions_batch[p] + 2ll * ((long long)env * Q.policy_size[p] + my_slot));
          act0 = v.x; act1 = v.y;
        }
      }
    }
    if (tid == 0 && tma_mask) {
      uint32_t total = 0;
#pragma unroll
      for (int q = 0; q < 2 * kMaxPolicies; q++)
        if (tma_mask & (1u << q)) total += prob_block(q).span;
      mbar_expect_tx(mbar, total);
#pragma unroll
      for (int p = 0; p < kMaxPolicies; p++) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const int q = 2 * p + h;
          if (tma_mask & (1u << q)) {
            const ProbBlock b = prob_block(q);
            const int np = Q.policy_size[p];
            const int A = h ? Q.A1 : Q.A0;
            const char *g = reinterpret_cast<const char *>(h ? Q.probs1[p] : Q.probs0[p]) +
                            4ll * env0 * np * A - b.lead;
            tma_load_1d(smem_u32(s_tile) + b.slot, g, b.span, mbar);
          }
        }
      }
    }
    griddep_launch_dependents();
  }

  if (tid < N) {
    stype[tid] = g_type;
    int rb = tid * F, rs = N * F;
    if (FUSED) {
#pragma unroll
      for (int p = 0; p < kMaxPolicies; p++)
        if (p == g_pol) { rb = tile_base(p) + g_slot * F; rs = Q.policy_size[p] * F; }
    }
    s_rowbase[tid] = rb;
    s_rowstride[tid] = rs;
  }
  if (tab_ok && tid < Q.A0 + Q.A1) s_tab[tid] = g_tab;
  if (tid < epb) s_nalive[tid] = 0;
  for (int i = tid; i < epb * (Ne - N); i += blockDim.x) {   // key padding: never a candidate
    const int e = i / (Ne - N), j = N + (i - e * (Ne - N));
    skx[e * Ne + j] = CUDART_INF_F;
    sky[e * Ne + j] = CUDART_INF_F;
  }
  if (active && a == 0) {
    const int t = g_t + 1;   // :391-393
    P.timestep[env] = t;
    s_t[le] = t;
    s_nrun[le] = g_nrun;
  }
  // s_nalive must be zero before the first atomicAdd of the kinematics (the fused variant
  // has its barrier in the sampling phase)
  if (!FUSED) __syncthreads();

  if (FUSED) {
    // random draw for both heads (independent of the probabilities: overlaps the copies)
    if (!ACTS_IN && active && !Q.uniforms) tc_draw_uniforms(Q, gi, rng_seed, rng_off, u0, u1);
    __syncthreads();                      // mbarrier initialised; tables / phase-0 arrays staged
    WDB_MARK(0)   // rng drawn, state requested
    if (tma_mask) mbar_wait(mbar, 0);      // TMA blocks landed
    WDB_MARK(1)   // probabilities landed
    if (ACTS_IN) {
      if (active) tc_push_actions(Q, gi, env, my_pol, 0, my_slot, act0, act1, false);
    } else if (active) {
      const int pol = my_pol, slot = my_slot;
      int np = 0, o0 = 0, o1 = 0;
      const float *g0 = nullptr, *g1 = nullptr;   // global rows of blocks that did not go by TMA
#pragma unroll
      for (int p = 0; p < kMaxPolicies; p++) {
        if (p == pol) {
          np = Q.policy_size[p];
          const ProbBlock b0 = prob_block(2 * p), b1 = prob_block(2 * p + 1);
          o0 = (int)((b0.slot + b0.lead) >> 2);      // float offset of the block's first row
          o1 = (int)((b1.slot + b1.lead) >> 2);
          const long long grow = (long long)env * np + slot;
          if (!(tma_mask & (1u << (2 * p)))) g0 = Q.probs0[p] + grow * Q.A0;
          if (!(tma_mask & (2u << (2 * p)))) g1 = Q.probs1[p] + grow * Q.A1;
        }
      }
      float *row0 = s_tile + o0 + (le * np + slot) * Q.A0;
      float *row1 = s_tile + o1 + (le * np + slot) * Q.A1;
      act0 = sample_row(row0, g0 ? g0 : row0, Q.A0, u0);
      act1 = sample_row(row1, g1 ? g1 : row1, Q.A1, u1);
      tc_push_actions(Q, gi, env, pol, np, slot, act0, act1);
    }
  } else if (active) {
    const int2 act = *reinterpret_cast<const int2 *>(P.actions + 2ll * gi);
    act0 = act.x; act1 = act.y;
  }

  WDB_MARK(2)   // actions sampled
  int alive = 0;
  if (active) {
    alive = st_alive;
    const TcMove mv = tc_move_agent(P, gi, st_x, st_y, st_sp, st_dir, st_acc, st_skill, alive,
                                    tab_ok ? s_tab[act0] : P.acc_actions[act0],
                                    tab_ok ? s_tab[Q.A0 + act1] : P.turn_actions[act1]);
    spos[li] = make_float2(mv.x, mv.y);
    skx[le * Ne + a] = alive ? mv.x : CUDART_INF_F;
    sky[le * Ne + a] = alive ? mv.y : CUDART_INF_F;
    ssp[li] = mv.sp; sacc[li] = mv.acc; sdir[li] = mv.dir;
    salive[li] = alive;
    if (alive) atomicAdd(&s_nalive[le], 1);
    // :283-291 reward initialisation (0 + edge + step), kept in shared memory so that tag
    // rewards can be accumulated atomically
    float r = 0.0f;
    if (alive) { r += mv.ep; r += P.step_rewards[a]; }
    srew[li] = r;
  }
  WDB_MARK(3)   // kinematics done
  __syncthreads();   // state staged; probability tile is dead from here on
  WDB_MARK(4)

  // tagger id list, built by warp 0
  if (warp == 0) {
    const int cnt = tc_build_tagger_list(stype, N, stag, lane);
    if (lane == 0) *s_ntag = cnt;
  }

  // ------------------------------------------------------------------ observations
  const double diag = sqrt(2.0) * L;                // :94
  const double inv_diag = 1.0 / diag;
  const float vnorm = P.max_speed + kEpsilon;       // :101
  const float two_pi = kTwoPi, inv_two_pi = 1.0f / kTwoPi;
  const int t_env = active ? s_t[le] : 0;
  const float2 *epos = spos + le * N;
  const int *ealive = salive + le * N;

  // bookkeeping words needed after the reward phase (loaded just before the feature phase)
  int done_prev = 0, steps_prev = 0;
  float run_prev = 0.0f;
  long long pi_slot = 0;
  auto load_bookkeeping = [&]() {
    if (FUSED && active) {
      done_prev = P.done[env];          // every thread: it derives the env's done flag itself
      if (a == 0 && Q.step_running_sum) steps_prev = Q.step_running_sum[env];
#pragma unroll
      for (int p = 0; p < kMaxPolicies; p++) {
        if (p == my_pol) {
          pi_slot = (long long)env * Q.policy_size[p] + my_slot;
          if (Q.reward_running_sum[p]) run_prev = Q.reward_running_sum[p][pi_slot];
        }
      }
    }
  };
  if (!P.use_full_obs) {
    uint32_t R[kListLen];
    int kk = 0;
    bool suspect = false;
    const uint32_t idmask = (1u << P.id_bits) - 1u;
    const bool net_ok = (K + 2 <= kListLen);
    if (active && alive) {
      const int nv = s_nalive[le] - 1;            // alive others
      kk = min(nv, K);
      if (net_ok) {
        // fast path: branch-free top-16 of packed (squared distance | id) keys.  Dead
        // agents sit at +inf and sort last; self has key (0 | a).
        const float2 pa = epos[a];
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
              const int b = min(max(pnr[p], 0), N - 1);
              if (b != a && ealive[b]) {
                const float2 pb = epos[b];
                tau = fmaxf(tau, sqdist(pa.x, pa.y, pb.x, pb.y));
                seen++;
              }
            }
          }
          // neighbours that left the game shrink the list: widen the disc accordingly
          if (seen < kk) tau *= 1.0f + 0.9f * (float)(kk - seen);
          if (seen == 0) tau = -1.0f;
          WDB_MARK(5)   // tau known
          uint32_t m0 = 0, m1 = 0, m2 = 0, m3 = 0;
          int cnt = 0;
          {
            const uint4 *kx4 = reinterpret_cast<const uint4 *>(kx);
            const uint4 *ky4 = reinterpret_cast<const uint4 *>(ky);
            // At most two passes: a list that came out too long (> kHistCap) or too short
            // (< kk + 1) is retried once with a smaller / larger disc before the sorting network
            // over all candidates has to run (any threshold is safe, see `hist_ok`).
#pragma unroll 1
            for (int pass = 0; pass < 2; pass++) {
              // mark with tau * (1 + 2^-17): everything left OUT of the mask is then farther
              // than m_out = that inflated threshold, which is the only thing the verification
              // needs to know about the rest (no running minimum inside the scan)
              const float tau_m = tau * 1.00000762939453125f;
              m0 = m1 = m2 = m3 = 0;
#define WDB_SCAN_WORD(W, M)                                                          \
              if (W * 32 < N) {                                                      \
                scan_16_nm<0>(M, kx4 + W * 8, ky4 + W * 8, pa.x, pa.y, tau_m);       \
                if (W * 32 + 16 < N)                                                 \
                  scan_16_nm<16>(M, kx4 + W * 8 + 4, ky4 + W * 8 + 4, pa.x, pa.y, tau_m); \
              }
              WDB_SCAN_WORD(0, m0) WDB_SCAN_WORD(1, m1) WDB_SCAN_WORD(2, m2) WDB_SCAN_WORD(3, m3)
#undef WDB_SCAN_WORD
              m_out = tau_m;
              cnt = __popc(m0) + __popc(m1) + __popc(m2) + __popc(m3);
              if (tau < 0.0f || (cnt >= kk + 1 && cnt <= kHistCap)) break;
              tau = (cnt > kHistCap) ? tau * (20.0f / (float)cnt) : tau * 2.5f;
            }
          }
          WDB_MARK(6)   // scan done
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
            {
              const int hbase = 0;
              WDB_REP16(WDB_HKEY)
              WDB_SORT16(c)
              r0 = c0; r1 = c1; r2 = c2; r3 = c3; r4 = c4; r5 = c5; r6 = c6; r7 = c7;
              r8 = c8; r9 = c9; r10 = c10; r11 = c11; r12 = c12; r13 = c13; r14 = c14;
              r15 = c15;
            }
            // candidates 17..32: inserted one at a time (see WDB_INSERT16)
#pragma unroll 1
            for (int e = kListLen; e < cnt; e++) {
              const int b = min((int)lst[e * kWarp], N - 1);
              const uint32_t key = (__float_as_uint(sqdist(pa.x, pa.y, kx[b], ky[b])) & ~idmask)
                                   | (uint32_t)b;
              WDB_INSERT16(r, key)
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
          network_top16(pa, kx, ky, N, idmask, out);
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
        if ((int)(R[0] & idmask) != a) suspect = true;     // a co-located agent sorted first
        float es[kListLen];
        bool misordered = false;
        {
          float prev = 0.0f;
#pragma unroll
          for (int i = 1; i < kListLen; i++) {
            es[i] = CUDART_INF_F;
            if (i <= m) {
              const float2 pb = epos[R[i] & idmask];
              es[i] = sqdist(pa.x, pa.y, pb.x, pb.y);
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
      } else {
        suspect = true;
      }
    }
    WDB_MARK(9)   // verified
    if (P.force_exact && active && alive) suspect = true;
    // exact path: the warp resolves its suspect agents one at a time, cooperatively
    unsigned todo = __ballot_sync(0xffffffffu, suspect);
    while (todo) {
      const int Lx = __ffs(todo) - 1;
      todo &= todo - 1;
      const int ax = __shfl_sync(0xffffffffu, a, Lx);
      const int lex = __shfl_sync(0xffffffffu, le, Lx);
      const int gix = __shfl_sync(0xffffffffu, gi, Lx);
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

    WDB_MARK(10)  // exact path done, ids stored
    // bookkeeping words needed after the reward phase: requested here, so that they are not
    // queued behind the burst of observation stores (kept out of the prologue: more live
    // registers across the neighbour search cost more than they save)
    load_bookkeeping();
    if (active) {
      float *orow = P.stage_obs ? (s_tile + s_rowbase[a] + le * s_rowstride[a])
                                : (P.obs + (long long)gi * F);
      // :121-139 zero-initialisation, restricted to what is not overwritten below
      if (!alive) {
        for (int f = 0; f < F; f++) orow[f] = 0.0f;
      } else {
        for (int p = kk; p < K; p++) {
#pragma unroll
          for (int f = 0; f < 7; f++) orow[f * K + p] = 0.0f;
        }
      }
      if (alive) {
        int *nn = P.nearest + (long long)gi * K;
        const float2 pa = epos[a];
        const float spa = ssp[li], acca = sacc[li], dira = sdir[li];
        const bool unit_v = (vnorm == 1.0f);
        const int *gids = (!net_ok && !P.scratch_in_smem)
                              ? P.g_nid + (long long)gi * (N - 1) : nullptr;
        // (x / vnorm with vnorm == 1.0f -- max_speed 1 -- is the identity: skipping the
        //  IEEE division also avoids its slow path, which a zero numerator always takes)
#define WDB_FEATURES(UNIT, UNROLL)                                                  \
        _Pragma(UNROLL)                                                             \
        for (int p = 0; p < kk; p++) {                                              \
          const int b = net_ok ? (int)idcol[p * kWarp] : gids[p];                   \
          nn[p] = b;                                            /* :202-211 */      \
          const int lb = le * N + b;                            /* :214-250 */      \
          const float2 pb = epos[b];                                                \
          orow[0 * K + p] = div_by_const_f64(pb.x - pa.x, diag, inv_diag);          \
          orow[1 * K + p] = div_by_const_f64(pb.y - pa.y, diag, inv_diag);          \
          const float dsp = ssp[lb] - spa, dac = sacc[lb] - acca;                   \
          orow[2 * K + p] = UNIT ? dsp : dsp / vnorm;                               \
          orow[3 * K + p] = UNIT ? dac : dac / vnorm;                               \
          orow[4 * K + p] = div_by_two_pi(sdir[lb] - dira, two_pi, inv_two_pi);     \
          orow[5 * K + p] = stype[b];                                               \
          orow[6 * K + p] = ealive[b];                                              \
        }
        if (unit_v) { WDB_FEATURES(true, "unroll 2") } else { WDB_FEATURES(false, "unroll 1") }
#undef WDB_FEATURES
        orow[7 * K] = static_cast<float>(t_env) / P.episode_length;   // :251-253
      }
    }
  } else {
    load_bookkeeping();
    // full observation (:55-113): one warp per row, lanes over the other agents, so every
    // feature plane of a row is written with unit-stride stores
    const int M = N - 1;
    const int rows = envs_here * N;
    for (int row = warp; row < rows; row += nwarps) {
      const int re = row / N, ra = row - re * N;
      const int renv = env0 + re;
      float *orow = P.obs ? P.obs + ((long long)renv * N + ra) * F : nullptr;
      float *orow2 = nullptr;
      if (FUSED) {
        const int pol = Q.agent_policy[ra];
#pragma unroll
        for (int p = 0; p < kMaxPolicies; p++)
          if (p == pol && Q.obs_next[p])
            orow2 = Q.obs_next[p] + ((long long)renv * Q.policy_size[p] + Q.agent_slot[ra]) * F;
      }
      const float2 *rpos = spos + re * N;
      const float *rsp = ssp + re * N, *racc = sacc + re * N, *rdir = sdir + re * N;
      const int *ral = salive + re * N;
      const bool self_alive = ral[ra] != 0;
      for (int idx = lane; idx < M; idx += kWarp) {
        const int b = idx < ra ? idx : idx + 1;
        float f0 = 0.f, f1 = 0.f, f2 = 0.f, f3 = 0.f, f4 = 0.f;
        if (self_alive) {
          f0 = div_by_const_f64(rpos[b].x - rpos[ra].x, diag, inv_diag);
          f1 = div_by_const_f64(rpos[b].y - rpos[ra].y, diag, inv_diag);
          f2 = static_cast<float>(rsp[b] - rsp[ra]) / vnorm;
          f3 = static_cast<float>(racc[b] - racc[ra]) / vnorm;
          f4 = div_by_two_pi(rdir[b] - rdir[ra], two_pi, inv_two_pi);
        }
        const float f5 = stype[b], f6 = ral[b];
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
        const float tt = self_alive ? static_cast<float>(s_t[re]) / P.episode_length : 0.0f;
        if (orow) orow[7 * M] = tt;
        if (orow2) orow2[7 * M] = tt;
      }
    }
  }
  // make the tile (written through the generic proxy) visible to the TMA engine
  WDB_MARK(11)  // features written
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();   // obs tile complete; srew initialised; tagger list ready
  WDB_MARK(12)

  // observation copy-out, part 1: every block of the tile whose shared / global addresses
  // and size are 16-byte aligned leaves through the TMA (cp.async.bulk), issued by one
  // thread now so that it overlaps the reward phase; the rest is copied by the threads at
  // the end of the kernel.
  if (!P.use_full_obs && P.stage_obs) {
    WDB_MARK(18)  // before the TMA store issue
    if (tid == 0 && out_mask) {
      if (out_mask & (1u << 8))
        tma_store_1d(P.obs + (long long)env0 * N * F, smem_u32(s_tile), 4u * envs_here * N * F);
#pragma unroll
      for (int p = 0; p < kMaxPolicies; p++) {
        if (FUSED && (out_mask & (1u << p))) {
          const int np = Q.policy_size[p];
          tma_store_1d(Q.obs_next[p] + (long long)env0 * np * F,
                       smem_u32(s_tile + tile_base(p)), 4u * envs_here * np * F);
        }
      }
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    WDB_MARK(19)  // TMA stores issued
  }
  // bf16 copy of the tile in the layout the next policy forward feeds to the tensor cores
  // (its fp32 obs path -- 4-byte loads of 284-byte rows, conversion, transposition -- is
  // the largest cost of that kernel; here the tile is in shared memory anyway).  Consecutive
  // threads take consecutive rows: conflict-free reads, 128-byte store segments.
  if (FUSED && !P.use_full_obs && P.stage_obs) {
    const int K1 = (F + 15) & ~15, nchunk = K1 / 8;
#pragma unroll
    for (int p = 0; p < kMaxPolicies; p++) {
      if (p < Q.n_policies && Q.obs_tiles[p]) {
        const int np = Q.policy_size[p], rows_p = envs_here * np;
        const float *blk = s_tile + tile_base(p);
        const long long grow0 = (long long)env0 * np;
        // (chunks that are all K padding stay zero from the allocation: never written)
        const int nreal = (F + 7) / 8;
        int c = tid / rows_p, lr = tid - c * rows_p;
        const int dc = blockDim.x / rows_p, dl = blockDim.x - dc * rows_p;
        for (int it = tid; it < rows_p * nreal; it += blockDim.x) {
          store_obs_chunk(Q.obs_tiles[p], grow0 + lr, c, K1, blk + lr * F, F);
          c += dc; lr += dl;
          if (lr >= rows_p) { lr -= rows_p; c++; }
        }
        (void)nchunk;
      }
    }
  }

  WDB_MARK(20)  // bookkeeping loads requested
  // ------------------------------------------------------------------ rewards / tags
  float r = active ? srew[li] : 0.0f;
  const bool is_runner = active && (stype[a] == 0);
  if (is_runner && alive) {                                  // :296-338
    const int tagger = tc_tagging_tagger(P, epos[a], epos, stag, *s_ntag);
    if (tagger >= 0) {
      r += P.tag_penalty;
      atomicAdd(&srew[le * N + tagger], P.tag_reward);
      if (P.runner_exits) {
        P.alive[gi] = 0;
        atomicSub(&s_nrun[le], 1);
      }
      if (P.stats) atomicAdd(&P.stats[1], 1);
    }
    if (t_env == P.episode_length) r += P.end_reward;        // :334-337
  }
  WDB_MARK(13)  // reward phase done
  __syncthreads();
  WDB_MARK(14)
  int done_now = 0;
  if (active) {
    r = (stype[a] == 1) ? srew[li] : r;
    P.rewards[gi] = r;
    const int nr = s_nrun[le];
    done_now = (t_env == P.episode_length || nr == 0) ? 1 : 0;   // :341-348
    if (a == 0) {
      P.num_runners[env] = nr;
      if (FUSED) s_done[le] = tc_book_env(P, Q, env, done_now, done_prev, steps_prev);
      else if (done_now) P.done[env] = 1;
    }
  }
  // every thread derives its env's done flag (no barrier: s_done is only for the reset phase,
  // which synchronises first)
  if (FUSED && active)
    tc_book_agent(Q, my_pol, pi_slot, r, run_prev, tc_sticky_done(done_now, done_prev));

  if (!P.use_full_obs && P.stage_obs) {
    // coalesced copy-out of the observation tile
    if (!FUSED) {
      if (!(out_mask & (1u << 8))) {
        const int total = envs_here * N * F;
        float *dst = P.obs + (long long)env0 * N * F;
        for (int i = tid; i < total; i += blockDim.x) dst[i] = s_tile[i];
      }
    } else {
#pragma unroll
      for (int p = 0; p < kMaxPolicies; p++) {
        if (p < Q.n_policies && Q.obs_next[p] && !(out_mask & (1u << p))) {
          // the tile block of policy p IS the [envs, Np, F] layout of obs_next[p]
          const int np = Q.policy_size[p];
          const int total = envs_here * np * F;
          const float *src = s_tile + tile_base(p);
          float *dst = Q.obs_next[p] + (long long)env0 * np * F;
          for (int i = tid; i < total; i += blockDim.x) dst[i] = src[i];
        }
      }
      if (P.obs) {
        // optional [E, N, F] `observations` array: one warp per agent row
        for (int e = 0; e < envs_here; e++) {
          for (int ra = warp; ra < N; ra += nwarps) {
            const float *src = s_tile + s_rowbase[ra] + e * s_rowstride[ra];
            float *dst = P.obs + ((long long)(env0 + e) * N + ra) * F;
            for (int f = lane; f < F; f += kWarp) dst[f] = src[f];
          }
        }
      }
    }
  }

  // the TMA stores must have read the tile (and, before the reset below overwrites the same
  // global rows for finished envs, must have completed) before the CTA goes on / exits
  WDB_MARK(15)  // bookkeeping + thread copy-out done
  if (tid == 0 && out_mask) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  WDB_MARK(16)  // TMA stores complete

  if (FUSED && Q.do_reset) {
    // done-masked reset of this CTA's envs (done / timestep already cleared above)
    __syncthreads();   // all global writes of this step by this CTA are issued
    for (int e = 0; e < envs_here; e++)
      if (s_done[e]) tc_reset_env<true>(Q, env0 + e, N, F, tid, blockDim.x, warp, nwarps, lane);
  }
  WDB_MARK(17)  // reset done
}

int g_tc_threads = 320; // wdb_set_option("tc_cta_threads", n): thread budget of one CTA (<= 320)

int g_tc_tail_split = 0;   // wdb_set_option("tc_tail_split", 0/1/2), off by default

// The packed kernel's geometry; shared-memory carve-up, must mirror the kernel prologue
int plan_packed(TcParams &P, const FusedParams *Q, TcPlan &plan) {
  const int N = P.N, K = P.K;
  const bool have_gscratch = P.g_nd && P.g_nid;
  const int n_envs = P.env_end - P.env_begin;   // the envs of this launch
  int epb = N >= g_tc_threads ? 1 : g_tc_threads / N;
  if (epb > n_envs) epb = n_envs;
  const int block = round_up(epb * N, 32);
  const int nwarps = block / 32;
  const int F = 7 * K + 1;
  const size_t base = tc_small_bytes(epb, N);
  // per-warp scratch: exact-path lists (8 B per agent) and/or the history byte list
  P.use_history = (g_tc_history && !P.use_full_obs && N <= 128 && K + 2 <= kListLen) ? 1 : 0;
  P.force_exact = g_tc_force_exact;
  size_t warp_bytes = 8ull * N;
  const size_t hist_bytes = (size_t)(kHistCap + 1) * kWarp;
  if (P.use_history && hist_bytes > warp_bytes) warp_bytes = hist_bytes;
  // sorted neighbour ids of every lane (uint16 columns) for the feature loop
  const size_t id_bytes = (!P.use_full_obs && K + 2 <= kListLen) ? (kListLen - 1) * kWarp * 2 : 0;
  if (id_bytes > warp_bytes) warp_bytes = id_bytes;
  warp_bytes = (warp_bytes + 15) & ~(size_t)15;
  const size_t scr = warp_bytes * nwarps;
  size_t tile_obs = P.use_full_obs ? 0 : sizeof(float) * (size_t)epb * N * F;
  size_t tile_probs = 0;   // (no probability tile when the actions come in sampled)
  if (Q && !Q->actions_in) {
    for (int p = 0; p < Q->n_policies; p++)
      tile_probs += ((sizeof(float) * (size_t)epb * Q->policy_size[p] * Q->A0 + 15) & ~(size_t)15) +
                    ((sizeof(float) * (size_t)epb * Q->policy_size[p] * Q->A1 + 15) & ~(size_t)15) + 64;
  }
  const size_t kMaxSmem = 200 * 1024;
  P.scratch_in_smem = (base + scr <= 64 * 1024) || !have_gscratch;
  if (P.scratch_in_smem && base + scr > kMaxSmem) return (int)cudaErrorInvalidValue;
  if (!P.scratch_in_smem) {
    warp_bytes = P.use_history ? ((hist_bytes + 15) & ~(size_t)15) : 0;
    if (id_bytes > warp_bytes) warp_bytes = id_bytes;
  }
  P.scr_warp_bytes = (int)warp_bytes;
  size_t smem = base + warp_bytes * nwarps;
  P.stage_obs = !P.use_full_obs && (smem + tile_obs <= 113 * 1024);   // two CTAs per SM
  size_t tile = P.stage_obs ? tile_obs : 0;
  if (tile_probs > tile) tile = tile_probs;
  smem += tile;
  if (smem > kMaxSmem) return (int)cudaErrorInvalidValue;
  if (!P.stage_obs && !P.use_full_obs && !P.obs) return (int)cudaErrorInvalidValue;
  P.epb = epb;
  int bits = 1;
  while ((1 << bits) < N) bits++;
  P.id_bits = bits;
  if (K + 2 > kListLen) {
    // selection falls back to the exact path for every agent; ids must survive until the
    // observation is written -> per-agent global scratch
    if (!have_gscratch) return (int)cudaErrorInvalidValue;
    P.scratch_in_smem = 0;
    P.scr_warp_bytes = 0;
    smem = base + tile;
  }
  plan.kernel = TcPlan::kPacked;
  plan.block = block;
  plan.grid = (n_envs + epb - 1) / epb;
  P.full_ctas = plan.grid;
  // Tail split (option, off): the kernel's time is waves x CTA latency.  When the last wave is
  // less than half full (not at config 2 on 132 SMs: 667 CTAs over 2 x 132 slots = 2 waves +
  // 139 CTAs), its envs go out as one-env CTAs instead: they start as the slots of the second wave free up and
  // spread over all SMs.  A one-env CTA's latency is the same dependent chain as a three-env
  // CTA's, so the last round barely shrinks.
  if (g_tc_tail_split == 2 && epb > 1 && plan.grid >= 2) {
    // test mode: half of the CTAs as one-env CTAs whatever the size
    const int full = plan.grid / 2;
    P.full_ctas = full;
    plan.grid = full + (n_envs - full * epb);
  } else if (g_tc_tail_split && epb > 1 && smem > 75 * 1024) {
    const int slots = 2 * kNumSMs;                    // two CTAs of this size per SM
    const int rem = plan.grid % slots;
    if (plan.grid > slots && rem > 0 && 2 * rem <= slots) {
      const int full = plan.grid - rem;
      const int tail_envs = n_envs - full * epb;
      P.full_ctas = full;
      plan.grid = full + tail_envs;
    }
  }
  plan.smem = smem;
  return 0;
}

template <bool FUSED, int MAXT, bool ACTS_IN = false>
int launch_t(const TcParams &P, const FusedParams &Q, const TcPlan &plan, cudaStream_t st) {
  static size_t configured = 0;
  if (plan.smem > 48 * 1024 && plan.smem > configured) {
    cudaError_t e = cudaFuncSetAttribute(tag_continuous_kernel<FUSED, MAXT, ACTS_IN>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)plan.smem);
    if (e != cudaSuccess) return (int)e;
    // all of the SM's unified L1 as shared memory: the CTAs are sized to fill it
    cudaFuncSetAttribute(tag_continuous_kernel<FUSED, MAXT, ACTS_IN>,
                         cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    configured = plan.smem;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)plan.grid, 1, 1);
  cfg.blockDim = dim3((unsigned)plan.block, 1, 1);
  cfg.dynamicSmemBytes = plan.smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = (FUSED && Q.pdl && g_pdl) ? 1 : 0;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, tag_continuous_kernel<FUSED, MAXT, ACTS_IN>, P, Q);
  if (e != cudaSuccess) return (int)e;
  return finish_launch();
}

// TcParams of one step of `e`, after the checks both entry points apply to it
int fill_params(TcParams &P, const wdb_tc_env &e) {
  if (!e.loc_x || !e.loc_y || !e.speed || !e.direction || !e.acceleration || !e.agent_types ||
      !e.edge_hit_reward_penalty || !e.acceleration_actions || !e.turn_actions ||
      !e.skill_levels || !e.still_in_the_game || !e.nearest_neighbor_ids || !e.rewards ||
      !e.step_rewards || !e.num_runners || !e.done || !e.env_timestep)
    return (int)cudaErrorInvalidValue;
  if (e.n_envs <= 0 || e.n_agents < 2 || e.n_agents > 4096 || e.num_other_agents_observed < 0)
    return (int)cudaErrorInvalidValue;
  P = {};
  P.n_envs = e.n_envs; P.N = e.n_agents; P.K = e.num_other_agents_observed;
  P.episode_length = e.episode_length;
  P.use_full_obs = e.use_full_observation; P.runner_exits = e.runner_exits_game_after_tagged;
  P.loc_x = e.loc_x; P.loc_y = e.loc_y; P.speed = e.speed; P.direction = e.direction;
  P.acceleration = e.acceleration; P.agent_types = e.agent_types;
  P.edge_pen = e.edge_hit_reward_penalty; P.edge_hit_penalty = e.edge_hit_penalty;
  P.grid_length = e.grid_length; P.acc_actions = e.acceleration_actions;
  P.turn_actions = e.turn_actions; P.max_speed = e.max_speed; P.skill = e.skill_levels;
  P.alive = e.still_in_the_game; P.obs = e.obs;
  P.g_nd = e.neighbor_distances; P.g_nid = e.neighbor_ids_sorted_by_distance;
  P.nearest = e.nearest_neighbor_ids; P.rewards = e.rewards; P.step_rewards = e.step_rewards;
  P.num_runners = e.num_runners; P.margin = e.distance_margin_for_reward;
  P.tag_reward = e.tag_reward_for_tagger; P.tag_penalty = e.tag_penalty_for_runner;
  P.end_reward = e.end_of_game_reward_for_runner; P.done = e.done;
  P.timestep = e.env_timestep; P.stats = e.stats;
  P.env_begin = 0; P.env_end = e.n_envs;
  return 0;
}

// Which kernel runs one TagContinuous step, with what geometry, or cudaErrorInvalidValue when
// none can.  Q is NULL for the env step alone; obs_next / obs_tiles: the fused step writes the
// next observations / their bf16 tiles for some policy.  Fills P's derived fields and `plan`;
// makes no CUDA call.
int tc_plan(TcParams &P, const FusedParams *Q, bool obs_next, bool obs_tiles, int blocks_per_env,
            TcPlan &plan) {
  plan = {};
  // blocks_per_env > 1: the env is spread over that many CTAs, launched as one thread-block
  // cluster (wdb_tc_wide.cu) -- the reference's multi-block mode, env_dim_mapper.h:22-31.
  // Observation tiles come from the packed kernel's staged tile only.
  // The actions-in mode (Q->actions_in) is a mode of the packed kernel alone: the
  // second-generation and cluster kernels always sample from the probabilities.
  const bool acts_in = Q && Q->actions_in;
  if (blocks_per_env > 1) {
    if (obs_tiles || acts_in) return (int)cudaErrorInvalidValue;
    return tc_wide_plan(P, Q, blocks_per_env, plan);
  }
  if (P.N > 1024) return (int)cudaErrorInvalidValue;   // one CTA per env: <= 1024 threads
  // envs too large for the packed kernel's shared-memory tile: the x-binned kernel with the
  // whole env in ONE CTA (a cluster of 1); wdb_set_option("tc_wide_single", 0) keeps the
  // first-generation single-CTA path for A/B runs
  if (g_tc_wide_single && P.N > 320 && !P.use_full_obs && P.K + 2 <= kListLen) {
    if (obs_tiles || acts_in) return (int)cudaErrorInvalidValue;
    return tc_wide_plan(P, Q, 1, plan);
  }
  if (tc_v2_eligible(P, Q, obs_tiles)) {
    if (acts_in) return (int)cudaErrorInvalidValue;
    return tc_v2_plan(P, plan);
  }
  const int err = plan_packed(P, Q, plan);
  if (err) return err;
  // the actions-in instance is built for the two-CTAs-per-SM geometry only
  if (acts_in && plan.block > 320) return (int)cudaErrorInvalidValue;
  // the per-policy observation push needs the shared-memory tile
  if (!P.stage_obs && !P.use_full_obs && (obs_next || obs_tiles))
    return (int)cudaErrorInvalidValue;
  if (P.use_full_obs && obs_tiles) return (int)cudaErrorInvalidValue;
  return 0;
}

int tc_launch(const TcParams &P, const FusedParams *Q, const TcPlan &plan, cudaStream_t st) {
  if (plan.kernel == TcPlan::kWide) return tc_wide_launch(P, Q, plan, st);
  if (plan.kernel == TcPlan::kV2) return tc_v2_launch(P, Q, plan, st);
  const FusedParams none = {};
  if (!Q)
    return plan.block <= 320 ? launch_t<false, 320>(P, none, plan, st)
                             : launch_t<false, 1024>(P, none, plan, st);
  if (Q->actions_in) return launch_t<true, 320, true>(P, *Q, plan, st);   // (tc_plan: block <= 320)
  return plan.block <= 320 ? launch_t<true, 320>(P, *Q, plan, st)
                           : launch_t<true, 1024>(P, *Q, plan, st);
}

// The rollout step's checks, in the order it applies them, then its plan.  shapes_only: no
// pointer of `ro` is checked, obs_next counts as written for every policy and the obs tiles
// as `with_tiles` says (wdb_tag_continuous_rollout_supported).
int plan_rollout(const wdb_tc_env *env, const wdb_tc_rollout *ro, bool shapes_only,
                 bool with_tiles, TcParams &P, FusedParams &Q, TcPlan &plan) {
  if (!env || !ro) return (int)cudaErrorInvalidValue;
  int err = fill_params(P, *env);
  if (err) return err;
  if (ro->n_policies < 1 || ro->n_policies > kMaxPolicies || ro->n_actions0 < 1 ||
      ro->n_actions1 < 1)
    return (int)cudaErrorInvalidValue;
  const bool acts_in = ro->actions_in != 0;
  if (!shapes_only) {
    if (!ro->agent_policy || !ro->agent_slot) return (int)cudaErrorInvalidValue;
    if (!acts_in && !ro->uniforms && !ro->rng_state) return (int)cudaErrorInvalidValue;
    if (ro->sampled_actions && ((uintptr_t)ro->sampled_actions & 7))
      return (int)cudaErrorMisalignedAddress;
  }
  Q = {};
  Q.rng = ro->rng_state; Q.uniforms = ro->uniforms;
  Q.n_policies = ro->n_policies; Q.A0 = ro->n_actions0; Q.A1 = ro->n_actions1;
  Q.agent_policy = ro->agent_policy; Q.agent_slot = ro->agent_slot;
  bool obs_next = shapes_only, obs_tiles = shapes_only && with_tiles;
  int total = 0;
  for (int p = 0; p < ro->n_policies; p++) {
    const wdb_tc_policy_io &io = ro->policy[p];
    if (io.n_agents < 1) return (int)cudaErrorInvalidValue;
    if (!shapes_only) {
      if (acts_in ? !io.actions_batch : (!io.probs0 || !io.probs1))
        return (int)cudaErrorInvalidValue;
      if (io.actions_batch && ((uintptr_t)io.actions_batch & 7))
        return (int)cudaErrorMisalignedAddress;
      if (io.obs_next_tiles && ((uintptr_t)io.obs_next_tiles & 15))
        return (int)cudaErrorMisalignedAddress;
      obs_next = obs_next || io.obs_next;
      obs_tiles = obs_tiles || io.obs_next_tiles;
    }
    Q.policy_size[p] = io.n_agents;
    Q.probs0[p] = io.probs0; Q.probs1[p] = io.probs1;
    Q.actions_batch[p] = io.actions_batch; Q.rewards_batch[p] = io.rewards_batch;
    Q.obs_next[p] = io.obs_next; Q.reward_running_sum[p] = io.reward_running_sum;
    Q.obs_tiles[p] = reinterpret_cast<unsigned char *>(io.obs_next_tiles);
    Q.episodic_reward_sum[p] = io.episodic_reward_sum;
    total += io.n_agents;
  }
  if (total != env->n_agents) return (int)cudaErrorInvalidValue;
  // a NULL actions_batch[0] disables the action push for every policy (kernel fast test)
  Q.actions_out = ro->sampled_actions;
  Q.actions_head0 = ro->sampled_actions_0; Q.actions_head1 = ro->sampled_actions_1;
  Q.done_batch = ro->done_batch; Q.step_running_sum = ro->step_running_sum;
  Q.episodic_step_sum = ro->episodic_step_sum; Q.num_completed = ro->num_completed_episodes;
  Q.reset_table = ro->reset_table; Q.n_reset = ro->n_reset_arrays;
  Q.obs_at_reset = ro->obs_at_reset; Q.do_reset = ro->reset_done_envs;
  Q.pdl = ro->launch_after_forward;
  Q.actions_in = acts_in;
  if (!shapes_only && Q.do_reset && Q.n_reset > 0 && !Q.reset_table)
    return (int)cudaErrorInvalidValue;
  // an env subrange: only the packed kernel takes one
  const int count = ro->env_count ? ro->env_count : env->n_envs - ro->env_begin;
  if (ro->env_begin < 0 || count < 1 || ro->env_begin + count > env->n_envs)
    return (int)cudaErrorInvalidValue;
  P.env_begin = ro->env_begin; P.env_end = ro->env_begin + count;
  err = tc_plan(P, &Q, obs_next, obs_tiles, env->blocks_per_env, plan);
  if (err) return err;
  if (count != env->n_envs && plan.kernel != TcPlan::kPacked) return (int)cudaErrorInvalidValue;
  return 0;
}

}  // namespace

namespace wdb {
int g_tc_wide_single = 1;  // wdb_set_option("tc_wide_single", 0/1)
int g_tc_history = 1;      // wdb_set_option("tc_history", 0/1)
int g_tc_force_exact = 0;  // wdb_set_option("tc_force_exact", 0/1)
}  // namespace wdb

extern int g_mlp_max_ctas;   // wdb_mlp.cu

WDB_API int wdb_set_option(const char *name, int value) {
  if (!name) return (int)cudaErrorInvalidValue;
  auto is = [&](const char *want) {
    int i = 0;
    for (; want[i] && name[i] == want[i]; i++) {}
    return !want[i] && !name[i];
  };
  if (is("tc_history")) { g_tc_history = value ? 1 : 0; return 0; }
  if (is("tc_force_exact")) { g_tc_force_exact = value ? 1 : 0; return 0; }
  if (is("tc_wide_single")) { g_tc_wide_single = value ? 1 : 0; return 0; }
  if (is("pdl")) { g_pdl = value ? 1 : 0; return 0; }
  if (is("tc_tail_split")) {
    if (value < 0 || value > 2) return (int)cudaErrorInvalidValue;
    g_tc_tail_split = value;
    return 0;
  }
  if (is("mlp_max_ctas")) {
    if (value < 0) return (int)cudaErrorInvalidValue;
    g_mlp_max_ctas = value;
    return 0;
  }
  {
    bool handled = false;
    int rc = tc_wide_set_option(name, value, &handled);
    if (handled) return rc;
    rc = tc_v2_set_option(name, value, &handled);
    if (handled) return rc;
  }
  if (is("tc_cta_threads")) {
    if (value < 32 || value > 320) return (int)cudaErrorInvalidValue;
    g_tc_threads = value;
    return 0;
  }
  return (int)cudaErrorInvalidValue;
}

WDB_API int wdb_tag_continuous_step(
    void *stream, int n_envs, int n_agents, int blocks_per_env, float *loc_x,
    float *loc_y, float *speed, float *direction, float *acceleration,
    const int *agent_types, float *edge_hit_reward_penalty, float edge_hit_penalty,
    float grid_length, const float *acceleration_actions, const float *turn_actions,
    float max_speed, int num_other_agents_observed, const float *skill_levels,
    int runner_exits_game_after_tagged, int *still_in_the_game,
    int use_full_observation, float *obs, const int *action_indices,
    float *neighbor_distances, int *neighbor_ids_sorted_by_distance,
    int *nearest_neighbor_ids, float *rewards, const float *step_rewards,
    int *num_runners, float distance_margin_for_reward, float tag_reward_for_tagger,
    float tag_penalty_for_runner, float end_of_game_reward_for_runner, int *done,
    int *env_timestep, int episode_length, int *stats) {
  if (blocks_per_env < 1) return (int)cudaErrorInvalidValue;
  const wdb_tc_env env = {   // in the field order of wdb_tc_env
      n_envs, n_agents, loc_x, loc_y, speed, direction, acceleration, agent_types,
      edge_hit_reward_penalty, edge_hit_penalty, grid_length, acceleration_actions,
      turn_actions, max_speed, num_other_agents_observed, skill_levels,
      runner_exits_game_after_tagged, still_in_the_game, use_full_observation, obs,
      neighbor_distances, neighbor_ids_sorted_by_distance, nearest_neighbor_ids, rewards,
      step_rewards, num_runners, distance_margin_for_reward, tag_reward_for_tagger,
      tag_penalty_for_runner, end_of_game_reward_for_runner, done, env_timestep,
      episode_length, stats, blocks_per_env};
  TcParams P;
  int err = fill_params(P, env);
  if (err) return err;
  if (!obs || !action_indices) return (int)cudaErrorInvalidValue;
  if ((uintptr_t)action_indices & 7) return (int)cudaErrorMisalignedAddress;
  P.actions = action_indices;
  TcPlan plan;
  err = tc_plan(P, nullptr, false, false, blocks_per_env, plan);
  if (err) return err;
  return tc_launch(P, nullptr, plan, as_stream(stream));
}

WDB_API int wdb_tag_continuous_rollout_step(void *stream, const wdb_tc_env *env,
                                            const wdb_tc_rollout *ro) {
  TcParams P;
  FusedParams Q;
  TcPlan plan;
  const int err = plan_rollout(env, ro, false, false, P, Q, plan);
  if (err) return err;
  return tc_launch(P, &Q, plan, as_stream(stream));
}

WDB_API int wdb_tag_continuous_rollout_supported(const wdb_tc_env *env,
                                                 const wdb_tc_rollout *ro, int with_obs_tiles) {
  TcParams P;
  FusedParams Q;
  TcPlan plan;
  return plan_rollout(env, ro, true, with_obs_tiles != 0, P, Q, plan);
}
