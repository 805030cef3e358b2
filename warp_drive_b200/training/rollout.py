"""RolloutEngine: the device-resident rollout loop
`policy forward -> sample -> env.step -> bookkeeping -> done-masked reset -> push to batch`.

This is the H100 re-design of TrainerBase._generate_rollout_batch and its helpers
(warp_drive/training/trainers/trainer_base.py:383-601, trainer_a2c.py:159-216): the
reference issues ~55 kernel launches and >= 5 host synchronisations per timestep
(SURVEY.md section 3.2); here one timestep has NO host synchronisation (done handling is
a device-side mask), and the whole T-step rollout is captured once in a CUDA graph and
replayed.
"""
import ctypes

import torch

from warp_drive_b200 import lib as _lib
from warp_drive_b200.utils.constants import Constants

_OBSERVATIONS = Constants.OBSERVATIONS
_ACTIONS = Constants.ACTIONS
_REWARDS = Constants.REWARDS
_DONE_FLAGS = Constants.DONE_FLAGS
_PROCESSED_OBSERVATIONS = Constants.PROCESSED_OBSERVATIONS
_ACTION_MASK = Constants.ACTION_MASK


class RolloutEngine:
    def __init__(self, env_wrapper, models, policy_tag_to_agent_id_map, sampler,
                 batch_size_per_env, use_cuda_graph=True, forward_dtype=None,
                 use_fused_step=True, write_observations=True, stats=None,
                 use_fused_forward=True, use_obs_tiles=False, use_pair_forward=False,
                 create_separate_placeholders_for_each_policy=False,
                 obs_dim_corresponding_to_num_agents="first", native_recurrent=True):
        self.env_wrapper = env_wrapper
        # heterogeneous agents: every policy steps through its own observations_{p}[_{key}],
        # sampled_actions[_{k}]_{p} and rewards_{p} arrays, and / or the env writes its
        # observations agent-last ([E, *F, N]); both are read by the fields gather
        self.separate = bool(create_separate_placeholders_for_each_policy)
        assert obs_dim_corresponding_to_num_agents in ("first", "last")
        self.agents_last = obs_dim_corresponding_to_num_agents == "last"
        self.use_pair_forward = bool(use_pair_forward)
        # A/B switch: with one forward launch per policy, launch the env step programmatically
        # dependent on the main-stream forward (option "pdl" must be on as well)
        self.pdl_after_fork = False
        self.dm = env_wrapper.cuda_data_manager
        self.models = models
        self.policy_map = policy_tag_to_agent_id_map
        self.policies = list(policy_tag_to_agent_id_map.keys())
        self.sampler = sampler
        self.T = int(batch_size_per_env)
        self.use_cuda_graph = use_cuda_graph
        self.forward_dtype = forward_dtype
        dev = self.dm.device
        self.E = env_wrapper.n_envs
        self.N = env_wrapper.n_agents
        self.ids = {p: torch.as_tensor(ids, dtype=torch.long, device=dev)
                    for p, ids in self.policy_map.items()}
        self.covers_all = {p: len(ids) == self.N and list(ids) == list(range(self.N))
                           for p, ids in self.policy_map.items()}
        from warp_drive_b200.training.utils.data_loader import (
            action_head_sizes, dict_observation_keys)

        # per policy: action heads, Dict observation keys (None for a Box space) and whether an
        # action mask rides along (a masked policy samples with the selection that never
        # returns a zero-probability action).  With shared placeholders every agent has the
        # same spaces, so these are the same for every policy.
        self.heads_of, self.continuous_of, self.obs_keys_of, self.masked_of = {}, {}, {}, {}
        for p, ids in self.policy_map.items():
            self.heads_of[p], self.continuous_of[p] = action_head_sizes(
                env_wrapper.env.action_space[ids[0]])
            self.obs_keys_of[p], self.masked_of[p] = dict_observation_keys(
                env_wrapper.env.observation_space[ids[0]])
            assert not (self.masked_of[p] and self.continuous_of[p]), (
                "an action mask needs discrete actions")
        p0 = self.policies[0]
        self.heads, self.obs_keys = self.heads_of[p0], self.obs_keys_of[p0]
        self.n_heads = len(self.heads)
        self.continuous = any(self.continuous_of.values())
        self.masked = any(self.masked_of.values())
        # diagonal Gaussian policies (FullyConnectedGaussian): forward -> [mean], sampled by
        # CUDASampler.sample_gaussian with the policy's log_std
        self.gaussian_of = {p: bool(getattr(models[p], "is_gaussian", False))
                            for p in self.policies}
        # tanh-squashed Gaussian actors (SAC; ActorAsPolicy of FullyConnectedSACActor): forward
        # -> [mu ++ raw log-std], sampled by CUDASampler.sample_squashed_gaussian
        self.squashed_of = {p: bool(getattr(models[p], "is_squashed_gaussian", False))
                            for p in self.policies}
        self.gaussian_of = {p: g or self.squashed_of[p] for p, g in self.gaussian_of.items()}
        self.gaussian = any(self.gaussian_of.values())
        assert self.separate or len(set(self.gaussian_of.values())) == 1, (
            "policies sharing the step placeholders are all Gaussian or none is")
        # Q networks (DQN's FullyConnectedQ): forward -> [Q values], sampled epsilon-greedily by
        # CUDASampler.sample_epsilon_greedy (sampler param `epsilon`, default 0: greedy), or in
        # the one-launch single-agent rollout by the same rule
        self.q_of = {p: bool(getattr(models[p], "is_q_network", False)) for p in self.policies}
        self.q_network = any(self.q_of.values())
        assert self.separate or len(set(self.q_of.values())) == 1, (
            "policies sharing the step placeholders are all Q networks or none is")
        # noisy Q networks (FullyConnectedQ with `noisy: true`): before each forward of the
        # per-step path, one wdb_noisy_draw launch per policy writes fresh factorized noise for
        # every env row, keyed by `noise_seed` (set by the trainer) and the policy's acting step
        # `acting_steps[p]`, a host counter.  DQN rollouts always pass sample params, so this path
        # runs eagerly and is never captured into a CUDA graph (rollout() does not capture a
        # noisy policy either).  The one-launch rollout's noisy Q kind draws the same noise from
        # the same key and advances the same counter.  Greedy steps (use_argmax) play the mean
        # network and draw nothing.
        self.noisy_of = {p: bool(getattr(models[p], "noisy", False)) for p in self.policies}
        self.noisy = any(self.noisy_of.values())
        self.noise_seed = 0
        self.acting_steps = {p: 0 for p in self.policies}
        self._acting_noise = {}
        # observations reach the policies through wdb_gather_policy_fields unless they are one
        # shared [E, N, F] Box array (wdb_gather_policy_rows)
        self.gather_fields = (self.separate or self.agents_last
                              or any(k is not None for k in self.obs_keys_of.values()))
        self.combined = None
        if len(self.policies) > 1 and not self.separate and not self.gaussian and not (
                self.q_network):
            self.combined = [torch.zeros((self.E, self.N, h), device=dev) for h in self.heads]
        # episodic statistics (device scalars: no host sync while rolling out)
        self.reward_running_sum = {p: torch.zeros((self.E, len(ids)), device=dev)
                                   for p, ids in self.policy_map.items()}
        self.step_running_sum = torch.zeros(self.E, dtype=torch.int32, device=dev)
        self.episodic_reward_sum = {p: torch.zeros((), device=dev) for p in self.policies}
        self.episodic_step_sum = torch.zeros((), dtype=torch.int64, device=dev)
        self.num_completed_episodes = torch.zeros((), dtype=torch.int64, device=dev)
        self._graph = None
        self._graph_stream = None
        # recurrent policies (FullyConnectedGRU): each keeps its agents' state hidden[p]
        # [E, Np, H] from step to step and rollout to rollout, and hidden_start[p], the state the
        # batch now in the *_batch* arrays started from (copied at t == 0 of every rollout,
        # inside the CUDA graph).  After every env step and its bookkeeping, ONE
        # wdb_recurrent_reset_done launch zeroes the rows of the envs that are done, before the
        # done-masked reset clears their flags: the step after an episode's end starts from zero
        # (FullyConnectedGRU.reset_hidden).  Their rollout forward is wdb_gru_policy_forward
        # where it takes the shape (native_recurrent), the model's torch step otherwise; a
        # recurrent Gaussian policy's forward gives its mean, sampled as any Gaussian policy's.
        self.recurrent_of = {p: bool(getattr(models[p], "is_recurrent", False))
                             for p in self.policies}
        self.recurrent = any(self.recurrent_of.values())
        self.hidden, self.hidden_start, self.native_gru = {}, {}, {}
        for p in self.policies:
            if self.recurrent_of[p]:
                shape = (self.E, len(self.policy_map[p]), int(models[p].hidden_size))
                self.hidden[p] = torch.zeros(shape, device=dev)
                self.hidden_start[p] = torch.zeros(shape, device=dev)
                if native_recurrent and forward_dtype is None:
                    from warp_drive_b200.training.models.fully_connected_gru import (
                        NativeGruStep)

                    if NativeGruStep.routed(models[p], self.E * len(self.policy_map[p])):
                        self.native_gru[p] = NativeGruStep(models[p])
        assert len(self.hidden) <= _lib.RECURRENT_MAX_POLICIES
        # (one [E, Np, A_k] buffer per softmax head, or a Gaussian policy's one mean [E, Np, A])
        self._recurrent_probs = {
            p: [torch.empty((self.E, len(self.policy_map[p]), h), device=dev)
                for h in models[p].output_dims] for p in self.native_gru}
        # ---- fused single-launch timestep (TagContinuous: 2 discrete heads, Box obs)
        self.fused = None
        if use_fused_step and self._fused_eligible():
            from warp_drive_b200.training.fused_tag_continuous import FusedTagContinuousStep

            self.fused = FusedTagContinuousStep(
                env_wrapper, self.policy_map, sampler, write_observations=write_observations,
                stats=stats)
            self.fused.set_bookkeeping(
                self.reward_running_sum, self.episodic_reward_sum, self.step_running_sum,
                self.episodic_step_sum, self.num_completed_episodes)
            obs = self._tensor(_OBSERVATIONS).view(self.E, self.N, -1)
            # observations of the *next* forward pass, per policy (filled by the kernel)
            self.cur_obs = {p: obs.index_select(1, self.ids[p]).contiguous()
                            for p in self.policies}

        # ---- whole-rollout single launch (single-agent classic control, small FullyConnected
        #      policy or actor)
        self.sa = None
        # (one agent: agent-last and agent-first observations are the same memory)
        if (use_fused_step and self.fused is None and not self.separate
                and (not self.agents_last or self.N == 1)):
            from warp_drive_b200.training.fused_single_agent import FusedSingleAgentRollout

            if (self.T >= 1
                    and FusedSingleAgentRollout.eligible(env_wrapper, models, self.policy_map)):
                p0 = self.policies[0]
                self.sa = FusedSingleAgentRollout(env_wrapper, models[p0], p0, sampler,
                                                  engine=self)
                self.sa.set_bookkeeping(
                    self.reward_running_sum, self.episodic_reward_sum, self.step_running_sum,
                    self.episodic_step_sum, self.num_completed_episodes)

        # ---- tensor-core forward (wgmma MLP kernel) for the fused path
        self.fused_forward = {}
        self._fwd_streams_of = {}     # per env group: the side streams of the smaller policies
        self.obs_tiles = {}
        self.sample_in_forward = False
        # (not for Q networks: that forward ends in a softmax)
        if (self.sa is None and use_fused_forward and forward_dtype is None and not self.continuous
                and not self.q_network):
            from warp_drive_b200.training.models.fused_forward import FusedPolicyForward

            # (also on the generic multi-launch path: gridworld, classic control with a policy
            #  too large for the whole-rollout kernel, envs with reset pools ...)
            if all(FusedPolicyForward.supported(m) for m in self.models.values()):
                self.fused_forward = {p: FusedPolicyForward(self.models[p]) for p in self.policies}
                self._probs = {p: [torch.empty((self.E, len(self.policy_map[p]), h), device=dev)
                                   for h in self.heads_of[p]] for p in self.policies}
                # bf16 MMA-ready mirror of the observations the next forward reads: written by
                # the fused env step itself (and by pack_obs whenever cur_obs changes outside it)
                # (off by default: at config 2 the env step's extra pass costs about what the
                #  forward saves)
                if (use_obs_tiles and self.fused is not None
                        and self.fused.eligible(env_wrapper, self.policy_map, obs_tiles=True)):
                    self.obs_tiles = {
                        p: torch.zeros(self.fused_forward[p].tiles_bytes(
                            self.E * len(self.policy_map[p])), dtype=torch.uint8, device=dev)
                        for p in self.policies}
                # The forwards also sample both heads, straight into the step's action batch
                # slot, and the fused step reads those actions instead of the probabilities
                # (no probability round trip, no sampling phase in the env kernel): when every
                # policy's shape samples and the step's launch plan takes its actions in.  The
                # same uniforms and CDF search, so the same actions as sampling in the step.
                self.sample_in_forward = (
                    self.fused is not None and not self.use_pair_forward
                    and all(f.samples for f in self.fused_forward.values())
                    and self.fused.eligible(env_wrapper, self.policy_map,
                                            obs_tiles=bool(self.obs_tiles), actions_in=True))
                if self.sample_in_forward:
                    self._agent_of_slot = {
                        p: torch.as_tensor(self.policy_map[p], dtype=torch.int32, device=dev)
                        for p in self.policies}
                    self._set_env_groups()

    def _set_env_groups(self, n_groups=None):
        """The sampling forward's schedule: the envs as one group, or as two halves that each
        run their own chain (forwards -> env step -> forwards ...) on their own streams, so one
        half's env step fills the SMs the other half's forwards leave idle (kernel tails,
        launch gaps).  Env replicas never interact, and every kernel indexes the shared arrays
        by global env, so both schedules compute the same bits.  Two groups when each half
        fills at least two env-step CTAs (a CTA carries up to 320 // N envs).  n_groups: force
        the count (tests and measurements compare the two schedules)."""
        per_cta = max(1, 320 // self.N)
        n = 2 if (not self.obs_tiles and self.E >= 4 * per_cta) else 1
        n = n if n_groups is None else n_groups
        half = self.E // 2
        self._groups = [(0, self.E)] if n == 1 else [(0, half), (half, self.E)]
        self._sampling = [
            {p: self.fused_forward[p].sampling(None, self._agent_of_slot[p], self.N,
                                               env_begin=e0) for p in self.policies}
            for e0, _ in self._groups]
        self._group_streams = [None] if n == 1 else [torch.cuda.Stream() for _ in self._groups]
        self._in_rollout = False
        self._graph = None

    def refresh_forward_weights(self):
        """Re-pack the policies' parameters for the tensor-core forward (after every
        optimizer step / checkpoint load)."""
        for fwd in self.fused_forward.values():
            fwd.refresh()

    def _fused_eligible(self):
        from warp_drive_b200.utils.spaces import Box, MultiDiscrete

        env = self.env_wrapper.env
        if self.separate or self.agents_last:
            return False
        if getattr(env, "name", "") != "TagContinuous" or len(self.policies) > 4:
            return False
        if self.continuous or self.n_heads != 2:
            return False
        if not isinstance(env.action_space[0], MultiDiscrete):
            return False
        if not isinstance(env.observation_space[0], Box):
            return False
        if self.T < 1 or self.dm.reset_target_to_pool:
            return False
        if any(getattr(m, "action_mask", None) is not None for m in self.models.values()):
            return False
        # its forwards keep no per-agent state
        if self.recurrent:
            return False
        # it samples its heads from softmax probabilities: a Q network acts epsilon-greedily
        if self.q_network:
            return False
        # its forwards read raw observations
        if any(getattr(m, "normalize_observations", False) for m in self.models.values()):
            return False
        # the library's launch plan decides the rest (shapes no kernel takes, e.g. envs too
        # large for the shared-memory observation tile, run the generic multi-launch path)
        from warp_drive_b200.training.fused_tag_continuous import FusedTagContinuousStep

        return FusedTagContinuousStep.eligible(self.env_wrapper, self.policy_map)

    def zero_hidden(self):
        """Restart every recurrent policy's state (all envs restarted)."""
        for h in self.hidden.values():
            h.zero_()

    def recurrent_reset_done(self):
        """Zero the recurrent states of every env whose _done_ is set: ONE launch for every
        recurrent policy (wdb_recurrent_reset_done)."""
        k = _lib.RecurrentReset()
        k.done = _lib.ptr(self._tensor("_done_"))
        k.n_envs, k.n_policies = self.E, len(self.hidden)
        for i, (p, h) in enumerate(self.hidden.items()):
            k.policy[i].hidden = _lib.ptr(h)
            k.policy[i].n_agents, k.policy[i].hidden_size = h.shape[1], h.shape[2]
        _lib.check(_lib.load().wdb_recurrent_reset_done(_lib.stream_ptr(), ctypes.byref(k)),
                   "recurrent_reset_done")

    def _recurrent_forward(self, p, obs_p):
        """Policy p's probabilities [per head] [E, Np, A_k] (a Gaussian policy: [mean
        [E, Np, A]]) from its observation rows, with its state hidden[p] advanced in place."""
        h = self.hidden[p]
        R = h.shape[0] * h.shape[1]
        obs = obs_p.reshape(R, -1)
        if p in self.native_gru:
            bufs = self._recurrent_probs[p]
            self.native_gru[p](obs, h, bufs)
            return bufs
        probs, h_new = self.models[p].step(obs, h.view(R, -1))
        h.copy_(h_new.view_as(h))
        return [q.view(h.shape[0], h.shape[1], -1) for q in probs]

    def resync_observations(self):
        """Re-gather the per-policy observation buffers from `observations` (call after
        anything outside the engine changed the env state, e.g. reset_all_envs); the recurrent
        policies' states restart."""
        self.zero_hidden()
        if self.fused is not None:
            obs = self._tensor(_OBSERVATIONS).view(self.E, self.N, -1)
            for p in self.policies:
                self.cur_obs[p].copy_(obs.index_select(1, self.ids[p]))
            self._repack_obs_tiles()

    def _repack_obs_tiles(self):
        if self.obs_tiles:
            for p in self.policies:
                self.fused_forward[p].pack_obs(self.cur_obs[p], self.obs_tiles[p])

    def materialize_observations(self):
        """Scatter the per-policy observation buffers back into the [E, N, F]
        `observations` array (only needed when the engine runs with
        write_observations=False and someone wants to read that array)."""
        if self.fused is not None:
            obs = self._tensor(_OBSERVATIONS).view(self.E, self.N, -1)
            for p in self.policies:
                obs.index_copy_(1, self.ids[p], self.cur_obs[p])

    def _forward(self, model, obs_p, mask=None):
        kw = {} if mask is None else {"action_mask": mask}
        if self.forward_dtype is not None:
            with torch.autocast("cuda", dtype=self.forward_dtype):
                probs, _ = model(obs_p, **kw)
            return [q.float().contiguous() for q in probs]
        probs, _ = model(obs_p, **kw)
        return [q.contiguous() for q in probs]

    def _forward_side_by_side(self, obs_in, probs, weights_stable=False, sampling=None,
                              group=0):
        """Every policy's fused forward, concurrently: the persistent MLP kernel uses one CTA
        per SM, so the SMs are split between the policies in proportion to their rows and the
        smaller policies run on side streams (fork/join by events, also under graph capture).
        Sequential launches would each pay the 195 KB weight load and leave most SMs idle
        during the small policy's single wave.  sampling: {policy: MlpSampling}, the forwards
        also sample (see sample_in_forward)."""
        if len(self.policies) == 1:
            self._one_forward(self.policies[0], obs_in, probs, sampling=sampling)
            return False
        if len(self.policies) == 2 and not self.obs_tiles and self.use_pair_forward:
            assert sampling is None, "the pair forward does not sample"
            # both policies in ONE launch (CTAs split by tile counts), no fork / join
            from warp_drive_b200.training.models.fused_forward import forward_pair

            pa, pb = sorted(self.policies,
                            key=lambda p: -(obs_in[p].numel() // obs_in[p].shape[-1]))
            forward_pair(self.fused_forward[pa], self.fused_forward[pb], obs_in[pa], obs_in[pb],
                         probs[pa], probs[pb], weights_stable=weights_stable)
            return True
        if not hasattr(self, "_fwd_plan"):
            n_sm = torch.cuda.get_device_properties(self.dm.device).multi_processor_count
            rows = {p: obs_in[p].numel() // obs_in[p].shape[-1] for p in self.policies}
            total = sum(rows.values())
            order = sorted(self.policies, key=lambda p: -rows[p])
            if len(order) == 2:
                # cost model in tile-times: ceil(tiles / SMs) + ~1.5 for the weight load;
                # pick the split that minimises the slower of the two
                tiles = {p: -(-rows[p] // 128) for p in order}
                best = None
                for k in range(1, n_sm // 2 + 1):
                    # (measured: the small policy's tiles run ~1.3x slower -- fewer CTAs share
                    #  its weights in L2 -- and a launch pays ~1.5 tile-times up front)
                    cost = max(-(-tiles[order[0]] // (n_sm - k)),
                               1.3 * -(-tiles[order[1]] // k)) + 1.5
                    if best is None or cost < best[0]:
                        best = (cost, k)
                share = {order[1]: best[1], order[0]: n_sm - best[1]}
            else:
                share = {p: max(1, min(n_sm - 1, -(-n_sm * rows[p] // total))) for p in order[1:]}
                share[order[0]] = max(1, n_sm - sum(share.values()))
            self._fwd_plan = (order, share)
        order, share = self._fwd_plan
        if group not in self._fwd_streams_of:
            self._fwd_streams_of[group] = [torch.cuda.Stream() for _ in order[1:]]
        cur = torch.cuda.current_stream()
        fork = torch.cuda.Event()
        fork.record(cur)
        joins = []
        for p, st in zip(order[1:], self._fwd_streams_of[group]):
            st.wait_event(fork)
            with torch.cuda.stream(st):
                self._one_forward(p, obs_in, probs, share[p], sampling)
                ev = torch.cuda.Event()
                ev.record(st)
            joins.append(ev)
        p = order[0]
        self._one_forward(p, obs_in, probs, share[p], sampling)
        for ev in joins:
            cur.wait_event(ev)
        return self.pdl_after_fork

    def _one_forward(self, p, obs_in, probs, max_ctas=0, sampling=None):
        smp = sampling[p] if sampling else None
        if self.obs_tiles:
            rows = obs_in[p].numel() // obs_in[p].shape[-1]
            self.fused_forward[p].forward_tiles(self.obs_tiles[p], rows, probs[p][0], probs[p][1],
                                                max_ctas=max_ctas, sampling=smp)
        else:
            self.fused_forward[p](obs_in[p], probs[p][0], probs[p][1], max_ctas=max_ctas,
                                  sampling=smp)

    def step_fused(self, t, uniforms=None):
        """One timestep = policy forwards + ONE libwdb200 launch."""
        with torch.no_grad():
            T = self.T
            if t >= 0:
                batches = {p: self._tensor(f"{_PROCESSED_OBSERVATIONS}_batch_{p}")
                           for p in self.policies}
                if t == 0 and not self.sample_in_forward:
                    for p in self.policies:
                        batches[p][0].copy_(self.cur_obs[p])
                obs_in = {p: batches[p][t] for p in self.policies}
                obs_next = {p: (batches[p][t + 1] if t + 1 < T else self.cur_obs[p])
                            for p in self.policies}
                actions_batch = {p: self._tensor(f"{_ACTIONS}_batch_{p}")[t]
                                 for p in self.policies}
                rewards_batch = {p: self._tensor(f"{_REWARDS}_batch_{p}")[t]
                                 for p in self.policies}
                done_batch = self._tensor(f"{_DONE_FLAGS}_batch")[t]
            else:   # evaluation-style step: no batch push
                obs_in = {p: self.cur_obs[p] for p in self.policies}
                if not hasattr(self, "_scratch_obs"):
                    self._scratch_obs = {p: torch.empty_like(self.cur_obs[p])
                                         for p in self.policies}
                obs_next = self._scratch_obs
                actions_batch = rewards_batch = done_batch = None
            if self.sample_in_forward:
                # the forwards sample into the batch slot (t < 0: into a scratch buffer), with
                # the RNG state the step would have sampled with
                if actions_batch is None:
                    if not hasattr(self, "_scratch_actions"):
                        self._scratch_actions = {
                            p: torch.empty((self.E, len(self.policy_map[p]), 2),
                                           dtype=torch.int32, device=self.dm.device)
                            for p in self.policies}
                    actions_batch = self._scratch_actions
                self._step_groups(t, obs_in, obs_next, actions_batch, rewards_batch, done_batch,
                                  uniforms)
            else:
                paired = False
                if self.fused_forward:
                    probs = self._probs
                    # t > 0: the kernel before this forward is the previous env step, not a
                    # weight re-pack -> the weight load may overlap its tail (programmatic launch)
                    paired = self._forward_side_by_side(obs_in, probs, weights_stable=t > 0)
                else:
                    probs = {p: self._forward(self.models[p], obs_in[p]) for p in self.policies}
                self.fused.launch(probs, actions_batch=actions_batch, rewards_batch=rewards_batch,
                                  obs_next=obs_next, done_batch=done_batch, uniforms=uniforms,
                                  obs_next_tiles=self.obs_tiles or None, after_forward=paired)
            if t < 0:
                for p in self.policies:
                    self.cur_obs[p].copy_(self._scratch_obs[p])

    def _step_groups(self, t, obs_in, obs_next, actions_batch, rewards_batch, done_batch,
                     uniforms):
        """One timestep of the sampling forwards and the env step, per env group on the
        group's stream.  Outside a rollout the groups fork from and join the current stream;
        inside one (_rollout_eager) they stay apart from the first step to the last."""
        cur = torch.cuda.current_stream()
        fork = not self._in_rollout and self._group_streams[0] is not None
        if fork:
            ev = torch.cuda.Event()
            ev.record(cur)
        for g, ((e0, e1), st) in enumerate(zip(self._groups, self._group_streams)):
            if fork:
                st.wait_event(ev)
            with torch.cuda.stream(st if st is not None else cur):
                if t == 0:
                    for p in self.policies:
                        obs_in[p][e0:e1].copy_(self.cur_obs[p][e0:e1])
                sampling = self._sampling[g]
                for p in self.policies:
                    s = sampling[p]
                    s.actions = _lib.ptr(actions_batch[p][e0:e1])
                    s.rng_state = self.fused.ro.rng_state
                    s.uniforms = _lib.ptr(uniforms)
                rows = {p: obs_in[p][e0:e1] for p in self.policies}
                probs = {p: [q[e0:e1] for q in self._probs[p]] for p in self.policies}
                # t > 0: the kernel before this forward is the previous env step, not a weight
                # re-pack -> the weight load may overlap its tail (programmatic launch)
                paired = self._forward_side_by_side(rows, probs, weights_stable=t > 0,
                                                    sampling=sampling, group=g)
                self.fused.launch(None, actions_batch=actions_batch, rewards_batch=rewards_batch,
                                  obs_next=obs_next, done_batch=done_batch, uniforms=uniforms,
                                  obs_next_tiles=self.obs_tiles or None, after_forward=paired,
                                  actions_in=True, envs=None if st is None else (e0, e1))
        if fork:
            self._join_groups(cur)

    def _join_groups(self, cur):
        for st in self._group_streams:
            ev = torch.cuda.Event()
            ev.record(st)
            cur.wait_event(ev)

    # ------------------------------------------------------------------ one timestep
    def _tensor(self, name):
        return self.dm.data_on_device_via_torch(name)

    def _slot(self, t):
        """Batch slot of timestep t of a rollout (t < 0: an evaluation step, no slot)."""
        return t

    # ---- native data movement of the generic path (csrc/wdb_rollout_generic.cu) ----------
    def _ids32(self, p):
        """int32 device copy of the policy's agent ids (None: the policy covers 0..N-1)."""
        if not hasattr(self, "_ids32_cache"):
            self._ids32_cache = {q: (None if self.covers_all[q]
                                     else self.ids[q].to(torch.int32).contiguous())
                                 for q in self.policies}
        return self._ids32_cache[p]

    def _move_rows(self, full, rows, scatter=False):
        """full [E, N, W] <-> rows {policy: [E, Np, W]} (4-byte elements), ONE launch for all
        policies in `rows` (wdb_gather_policy_rows)."""
        assert full.is_contiguous() and full.element_size() == 4
        g = _lib.Gather()
        g.n_envs, g.n_agents = self.E, self.N
        g.width = full.numel() // (self.E * self.N)
        g.n_policies, g.scatter = len(rows), int(bool(scatter))
        g.full = _lib.ptr(full)
        for i, (p, r) in enumerate(rows.items()):
            assert r.is_contiguous() and r.element_size() == 4
            assert r.numel() == self.E * len(self.policy_map[p]) * g.width, (p, r.shape)
            io = g.policy[i]
            io.n_agents = len(self.policy_map[p])
            io.agent_ids = _lib.ptr(self._ids32(p))
            io.rows = _lib.ptr(r)
        _lib.check(_lib.load().wdb_gather_policy_rows(_lib.stream_ptr(), ctypes.byref(g)),
                   "gather_policy_rows")

    def _field_plan(self):
        """The fields wdb_gather_policy_fields moves: (source, width, destination, column,
        index of the policy whose own array it is or None) per key, and per policy the widths
        (F_p, sum of its head sizes) of its two destinations."""
        if not hasattr(self, "_fields"):
            owners = (list(enumerate(self.policies)) if self.separate
                      else [(None, self.policies[0])])
            fields = []
            for i, p in owners:
                prefix = f"{_OBSERVATIONS}_{p}" if self.separate else _OBSERVATIONS
                n_src = len(self.policy_map[p]) if self.separate else self.N
                keys = self.obs_keys_of[p]
                names = ([(prefix, False)] if keys is None
                         else [(f"{prefix}_{k}", False) for k in keys])
                if self.masked_of[p]:
                    names.append((f"{prefix}_{_ACTION_MASK}", True))
                col = 0
                for name, is_mask in names:
                    src = self._tensor(name)
                    assert src.dtype in (torch.float32, torch.int32), (
                        f"observation array {name!r}: only float32 / int32 arrays are gathered")
                    assert src.is_contiguous()
                    width = src.numel() // (self.E * n_src)
                    if is_mask:
                        assert width == sum(self.heads_of[p]), (
                            "action_mask must cover every head's actions")
                        fields.append((src, width, 1, 0, i))
                    else:
                        fields.append((src, width, 0, col, i))
                        col += width
            assert len(fields) <= _lib.GATHER_MAX_FIELDS
            widths = {p: (self._tensor(f"{_PROCESSED_OBSERVATIONS}_batch_{p}").shape[-1],
                          sum(self.heads_of[p])) for p in self.policies}
            for src, width, dst, col, i in fields:
                owned = self.policies if i is None else [self.policies[i]]
                assert all(col + width <= widths[p][dst] for p in owned), (
                    "observation widths differ from the processed observation batch")
            self._fields = (fields, widths)
        return self._fields

    def _gather_fields(self, obs_rows, mask_rows):
        """Every observation array of every policy -> obs_rows {policy: [E, Np, F_p]} (the
        non-mask keys concatenated, converted to float32) and its action mask -> mask_rows
        {policy: [E, Np, sum A_p]}, ONE launch for all policies (wdb_gather_policy_fields).
        Sources are the shared [E, N, ...] arrays or, with separate placeholders, each
        policy's own [E, Np, ...] ones; agent-last sources ([E, *F, Ns]) are transposed on
        the way."""
        fields, widths = self._field_plan()
        p0 = self.policies[0]
        g = _lib.GatherFields()
        g.n_envs, g.n_agents = self.E, self.N
        g.n_policies, g.n_fields = len(self.policies), len(fields)
        g.dst_width[0], g.dst_width[1] = widths[p0]
        for j, (src, width, dst, col, i) in enumerate(fields):
            f = g.field[j]
            f.src, f.width, f.is_int32 = _lib.ptr(src), width, int(src.dtype == torch.int32)
            f.dst, f.col = dst, col
            f.policy_mask, f.own_rows = (0, 0) if i is None else (1 << i, 1)
            f.agents_last = int(self.agents_last)
        for i, p in enumerate(self.policies):
            io = g.policy[i]
            io.n_agents = len(self.policy_map[p])
            io.agent_ids = None if self.separate else _lib.ptr(self._ids32(p))
            io.rows[0] = _lib.ptr(obs_rows[p])
            io.rows[1] = _lib.ptr(mask_rows[p]) if mask_rows[p] is not None else None
            io.dst_width[0], io.dst_width[1] = widths[p]
        _lib.check(_lib.load().wdb_gather_policy_fields(_lib.stream_ptr(), ctypes.byref(g)),
                   "gather_policy_fields")

    def evaluate_policies(self, t):
        """obs -> per-head probabilities [E, N, A_k] (trainer_a2c.py:159-216).  The per-policy
        observation rows go to the batch slot in one gather launch and the forward reads the
        slot; the per-policy probabilities return to the sampler's [E, N, A] arrays in one
        scatter launch per head.  With separate placeholders: {policy: per-head probabilities
        [E, Np, A_k]}, which the sampler reads as they are; so with several Gaussian policies
        ({policy: [mean [E, Np, A]]})."""
        mask_p = {p: None for p in self.policies}
        if self.gather_fields:
            obs_p, mask_p = self._field_slots(t)
        elif t >= 0:
            obs = self._tensor(_OBSERVATIONS).view(self.E, self.N, -1)
            s = self._slot(t)
            obs_p = {p: self._tensor(f"{_PROCESSED_OBSERVATIONS}_batch_{p}")[s]
                     for p in self.policies}
            self._move_rows(obs, obs_p)
        else:
            obs = self._tensor(_OBSERVATIONS).view(self.E, self.N, -1)
            if not hasattr(self, "_obs_scratch"):
                self._obs_scratch = {
                    p: torch.empty((self.E, len(self.policy_map[p]), obs.shape[-1]),
                                   dtype=obs.dtype, device=obs.device)
                    for p in self.policies if not self.covers_all[p]}
            obs_p = {p: obs for p in self.policies if self.covers_all[p]}
            obs_p.update(self._obs_scratch)
            if self._obs_scratch:
                self._move_rows(obs, self._obs_scratch)
        # a Q network's forward leaves its outputs raw: the epsilon-greedy sampler applies the
        # step's mask rows (sample_actions)
        self._q_masks = mask_p
        per_policy = {}
        for p in self.policies:
            if self.recurrent_of[p]:
                per_policy[p] = self._recurrent_forward(p, obs_p[p])
            elif self.fused_forward:
                # wgmma forward straight into the persistent probability buffers
                bufs = self._probs[p]
                self.fused_forward[p](obs_p[p], bufs[0], bufs[1] if len(bufs) > 1 else None,
                                      mask=mask_p[p])
                per_policy[p] = bufs
            else:
                per_policy[p] = self._forward(self.models[p], obs_p[p].view(
                    self.E, len(self.policy_map[p]), -1), mask_p[p])
        if self.separate or ((self.gaussian or self.q_network) and len(self.policies) > 1):
            return per_policy
        if self.combined is None:
            return per_policy[self.policies[0]]
        for k in range(self.n_heads):
            self._move_rows(self.combined[k], {p: per_policy[p][k] for p in self.policies},
                            scatter=True)
        return self.combined

    def _field_slots(self, t):
        """Per-policy observation and mask rows for timestep t, filled by one gather launch:
        the batch slots of t (t >= 0), or scratch rows (an evaluation step)."""
        if t >= 0:
            s = self._slot(t)
            obs_p = {p: self._tensor(f"{_PROCESSED_OBSERVATIONS}_batch_{p}")[s]
                     for p in self.policies}
            mask_p = {p: (self._tensor(f"{_ACTION_MASK}_batch_{p}")[s] if self.masked_of[p]
                          else None) for p in self.policies}
        else:
            if not hasattr(self, "_field_scratch"):
                dev = self.dm.device
                _, widths = self._field_plan()
                self._field_scratch = (
                    {p: torch.empty((self.E, len(self.policy_map[p]), widths[p][0]), device=dev)
                     for p in self.policies},
                    {p: (torch.empty((self.E, len(self.policy_map[p]), widths[p][1]),
                                     device=dev) if self.masked_of[p] else None)
                     for p in self.policies})
            obs_p, mask_p = self._field_scratch
        self._gather_fields(obs_p, mask_p)
        return obs_p, mask_p

    def _sample(self, probs, suffix, heads, masked, sample_params):
        """probs [per head] -> sampled_actions{suffix} (one head) or sampled_actions_{k}{suffix},
        combined into sampled_actions{suffix} (several)."""
        dm = self.dm
        if masked:
            sample_params = dict(sample_params, nonzero=True)
        if len(heads) == 1:
            self.sampler.sample(dm, probs[0], f"{_ACTIONS}{suffix}", write_cum_distr=False,
                                **sample_params)
        else:
            actions = self._tensor(f"{_ACTIONS}{suffix}")
            for k in range(len(heads)):
                self.sampler.sample(dm, probs[k], f"{_ACTIONS}_{k}{suffix}",
                                    write_cum_distr=False,
                                    combined=(actions, len(heads), k), **sample_params)

    def _sample_gaussian(self, means, suffix, sample_params):
        """{policy: mean [E, Np, A]} -> sampled_actions{suffix} [E, N, A] (and the per-dimension
        sampled_actions_{k}{suffix} when A > 1).  One policy covering the array samples into it
        directly; several policies sharing it sample their own rows, which one launch then
        scatters into place."""
        actions = self._tensor(f"{_ACTIONS}{suffix}")
        if len(means) == 1:
            (p, mean), = means.items()
            self._draw_gaussian(p, mean, actions, sample_params)
        else:
            if not hasattr(self, "_gaussian_rows"):
                self._gaussian_rows = {p: m.new_empty(m.shape[:-1] + actions.shape[-1:])
                                       for p, m in means.items()}
            for p, mean in means.items():
                self._draw_gaussian(p, mean, self._gaussian_rows[p], sample_params)
            self._move_rows(actions, self._gaussian_rows, scatter=True)
        if actions.shape[-1] > 1:
            for k in range(actions.shape[-1]):
                self._tensor(f"{_ACTIONS}_{k}{suffix}").copy_(actions[..., k:k + 1])

    def _draw_gaussian(self, p, head, out, sample_params):
        """Policy p's Gaussian actions into `out` [E, Np, A]: a diagonal Gaussian's head is the
        mean, a squashed Gaussian's is [mu ++ raw log-std]."""
        if self.squashed_of[p]:
            actor = self.models[p].actor
            self.sampler.sample_squashed_gaussian(
                head, out, actor.action_scale, actor.action_bias, actor.log_std_min,
                actor.log_std_max, **sample_params)
        else:
            self.sampler.sample_gaussian(head, self.models[p].log_std, out, **sample_params)

    def _sample_epsilon_greedy(self, q_values, suffix, sample_params):
        """{policy: Q values [E, Np, A]} -> sampled_actions{suffix} [E, N, 1] int32, as
        _sample_gaussian: one policy covering the array samples into it, several sample their
        own rows, which one launch scatters into place.  A masked policy samples over the valid
        actions of the mask rows its last evaluate_policies gathered (the batch slot, or the
        scratch rows of an evaluation step).  A branching Q network of D > 1 heads samples
        each head on its own into [E, Np, D] rows (and the per-head sampled_actions_{k}{suffix}
        are written as well)."""
        actions = self._tensor(f"{_ACTIONS}{suffix}")
        masks = getattr(self, "_q_masks", {})

        def draw(p, q, out):
            sizes = getattr(self.models[p], "branch_sizes", None)
            kw = {"branch_sizes": sizes} if sizes is not None and len(sizes) > 1 else {
                "action_mask": masks.get(p)}
            self.sampler.sample_epsilon_greedy(q, out, **kw, **sample_params)
        if len(q_values) == 1:
            (p, q), = q_values.items()
            draw(p, q, actions)
        else:
            if not hasattr(self, "_q_rows"):
                self._q_rows = {p: torch.empty(q.shape[:-1] + actions.shape[-1:],
                                               dtype=torch.int32, device=q.device)
                                for p, q in q_values.items()}
            for p, q in q_values.items():
                draw(p, q, self._q_rows[p])
            self._move_rows(actions, self._q_rows, scatter=True)
        if actions.shape[-1] > 1:
            for k in range(actions.shape[-1]):
                self._tensor(f"{_ACTIONS}_{k}{suffix}").copy_(actions[..., k:k + 1])

    def sample_actions(self, probs, t, **sample_params):
        """probs -> sampled_actions (trainer_base.py:466-512); the per-policy batch push of the
        actions happens in bookkeep().  With separate placeholders, each policy's
        probabilities go to its own sampled_actions[_{k}]_{p}."""
        if self.separate:
            for p in self.policies:
                if self.gaussian_of[p]:
                    self._sample_gaussian({p: probs[p][0]}, f"_{p}", sample_params)
                elif self.q_of[p]:
                    self._sample_epsilon_greedy({p: probs[p][0]}, f"_{p}", sample_params)
                else:
                    self._sample(probs[p], f"_{p}", self.heads_of[p], self.masked_of[p],
                                 sample_params)
        elif self.q_network:
            q = ({p: v[0] for p, v in probs.items()} if isinstance(probs, dict)
                 else {self.policies[0]: probs[0]})
            self._sample_epsilon_greedy(q, "", sample_params)
        elif self.gaussian:
            means = ({p: q[0] for p, q in probs.items()} if isinstance(probs, dict)
                     else {self.policies[0]: probs[0]})
            self._sample_gaussian(means, "", sample_params)
        else:
            self._sample(probs, "", self.heads, self.masked, sample_params)

    def bookkeep(self, t):
        """done / rewards / actions -> batches, running episodic sums: ONE launch
        (wdb_rollout_bookkeep), no host synchronisation (trainer_base.py:514-601 uses
        nonzero() / len())."""
        s = self._slot(t)
        k = _lib.Bookkeep()
        k.n_envs, k.n_agents, k.n_policies = self.E, self.N, len(self.policies)
        k.done = _lib.ptr(self._tensor("_done_"))
        if self.separate:
            k.n_heads = 0
        else:
            actions = (self._tensor(_ACTIONS) if self.dm.is_data_on_device_via_torch(_ACTIONS)
                       else None)
            k.n_heads = (actions.numel() // (self.E * self.N)) if actions is not None else 0
            k.rewards = _lib.ptr(self._tensor(_REWARDS))
            k.actions = _lib.ptr(actions)
        k.done_batch = _lib.ptr(self._tensor(f"{_DONE_FLAGS}_batch")[s]) if t >= 0 else None
        k.step_running_sum = _lib.ptr(self.step_running_sum)
        k.episodic_step_sum = _lib.ptr(self.episodic_step_sum)
        k.num_completed_episodes = _lib.ptr(self.num_completed_episodes)
        for i, p in enumerate(self.policies):
            io = k.policy[i]
            io.n_agents = len(self.policy_map[p])
            if self.separate:
                own = self._tensor(f"{_ACTIONS}_{p}")
                io.rewards = _lib.ptr(self._tensor(f"{_REWARDS}_{p}"))
                io.actions = _lib.ptr(own)
                io.n_heads = own.numel() // (self.E * io.n_agents)
                has_actions = True
            else:
                io.agent_ids = _lib.ptr(self._ids32(p))
                has_actions = actions is not None
            if t >= 0:
                io.rewards_batch = _lib.ptr(self._tensor(f"{_REWARDS}_batch_{p}")[s])
                if has_actions:
                    io.actions_batch = _lib.ptr(self._tensor(f"{_ACTIONS}_batch_{p}")[s])
            io.reward_running_sum = _lib.ptr(self.reward_running_sum[p])
            io.episodic_reward_sum = _lib.ptr(self.episodic_reward_sum[p])
        _lib.check(_lib.load().wdb_rollout_bookkeep(_lib.stream_ptr(), ctypes.byref(k)),
                   "rollout_bookkeep")

    def policy_step_arrays(self, p):
        """(rewards [E, Np], sampled actions [E, Np, n_heads]) of policy p's agents."""
        if self.separate:
            return self._tensor(f"{_REWARDS}_{p}"), self._tensor(f"{_ACTIONS}_{p}")
        rewards, actions = self._tensor(_REWARDS), self._tensor(_ACTIONS)
        if self.covers_all[p]:
            return rewards, actions
        return rewards.index_select(1, self.ids[p]), actions.index_select(1, self.ids[p])

    def bookkeep_torch(self, t):
        """The same bookkeeping in plain torch ops (the parity reference of bookkeep() in
        tests/test_gpu_rollout.py; not used by the engine)."""
        raw_done = self._tensor("_done_")
        if t >= 0:
            self._tensor(f"{_DONE_FLAGS}_batch")[t].copy_(raw_done)
        done = (raw_done > 0).to(torch.int32)
        donef = done.to(torch.float32)
        for p in self.policies:
            r_p, a_p = self.policy_step_arrays(p)
            if t >= 0:
                self._tensor(f"{_ACTIONS}_batch_{p}")[t].copy_(a_p)
                self._tensor(f"{_REWARDS}_batch_{p}")[t].copy_(r_p)
            run = self.reward_running_sum[p]
            run.add_(r_p)
            self.episodic_reward_sum[p].add_((run * donef[:, None]).sum())
            run.mul_(1.0 - donef[:, None])
        self.step_running_sum.add_(1)
        self.episodic_step_sum.add_((self.step_running_sum * done).sum())
        self.step_running_sum.mul_(1 - done)
        self.num_completed_episodes.add_(done.sum())

    def _set_acting_noise(self):
        """Fresh per-row noise for every noisy policy's head (one launch each), set on its
        NoisyLinear layers; returns the layers."""
        from warp_drive_b200.training.algorithms.fused_dqn import NOISY_ACTING, draw_noise

        layers = []
        for p in self.policies:
            if not self.noisy_of[p]:
                continue
            model = self.models[p]
            noisy = model.noisy_layers()
            if p not in self._acting_noise:
                rows = self.E * len(self.policy_map[p])
                dev = self.dm.device
                self._acting_noise[p] = [
                    (torch.empty(rows, L.in_features, device=dev),
                     torch.empty(rows, L.out_features, device=dev)) for L in noisy]
            draw_noise(model, self.noise_seed, NOISY_ACTING, self.acting_steps[p],
                       rows=self._acting_noise[p])
            self.acting_steps[p] += 1
            for L, pair in zip(noisy, self._acting_noise[p]):
                L.noise = pair
            layers += noisy
        return layers

    def step(self, t, **sample_params):
        if self.fused is not None and not sample_params:
            return self.step_fused(t)
        if self.sa is not None and self._sa_params_ok(sample_params):
            with torch.no_grad():
                self.sa.launch(1, t0=max(self._slot(t), 0), record=t >= 0, **sample_params)
            return None
        greedy = False
        if self.q_network:                     # use_argmax: the mean network, epsilon 0
            greedy = bool(sample_params.pop("use_argmax", False))
            if greedy:
                sample_params["epsilon"] = 0.0
        with torch.no_grad():
            if self.recurrent and t == 0:
                for p, h in self.hidden.items():
                    self.hidden_start[p].copy_(h)
            noisy = self._set_acting_noise() if self.noisy and not greedy else []
            try:
                probs = self.evaluate_policies(t)
            finally:
                for L in noisy:
                    L.noise = None
            self.sample_actions(probs, t, **sample_params)
            self.env_wrapper.step_all_envs()
            self.bookkeep(t)
            if self.recurrent:
                self.recurrent_reset_done()
            # done-masked reset: a no-op for envs that are not done, so no host-side
            # `if done_flags.any()` (trainer_base.py:421-422) is needed
            self.env_wrapper.reset_only_done_envs()

    # ------------------------------------------------------------------ T-step rollout
    def _rollout_eager(self, **sample_params):
        groups = (self.fused is not None and self.sample_in_forward and not sample_params
                  and self._group_streams[0] is not None)
        if not groups:
            for t in range(self.T):
                self.step(t, **sample_params)
            return
        # the env groups run apart for the whole rollout: fork once, join once
        cur = torch.cuda.current_stream()
        ev = torch.cuda.Event()
        ev.record(cur)
        for st in self._group_streams:
            st.wait_event(ev)
        self._in_rollout = True
        try:
            for t in range(self.T):
                self.step(t)
        finally:
            self._in_rollout = False
            self._join_groups(cur)

    def _sa_params_ok(self, sample_params):
        """The whole-rollout kernel takes the categorical sampler's argmax switch, or the OU
        parameters of a continuous action (the other sampler arguments are test hooks)."""
        allowed = (("damping", "stddev", "scale") if self.continuous and not self.gaussian
                   else ("epsilon", "use_argmax") if self.q_network else ("use_argmax",))
        return all(k in allowed for k in sample_params)

    def rollout(self, **sample_params):
        """Generate one training batch (T timesteps for every env replica)."""
        if self.sa is not None and self._sa_params_ok(sample_params):
            # ONE launch for all T timesteps (no CUDA graph needed)
            with torch.no_grad():
                self.sa.launch(self.T, t0=0, record=True, **sample_params)
            return
        if not self.use_cuda_graph or sample_params or self.noisy:
            self._rollout_eager(**sample_params)
            return
        if self._graph is None:
            # warm-up on a side stream (cuBLAS workspaces, lazy inits), then capture
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                # an evaluation-style step: advances the envs AND the engine's current
                # observations consistently, records nothing (a step(0) here would leave
                # cur_obs one state behind the env for the first captured transition)
                self.step(-1)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                self._rollout_eager()
            self._graph = graph
        self._graph.replay()
