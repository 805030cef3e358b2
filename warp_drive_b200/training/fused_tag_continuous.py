"""Host-side binding of wdb_tag_continuous_rollout_step: ONE kernel launch per rollout
timestep of TagContinuous (sample both heads -> env step -> push actions / rewards / done /
next observations -> episodic sums -> done-masked reset).

The structs are filled once from the data manager (device pointers are stable), only the
per-timestep batch-slot pointers change between launches.
"""
import ctypes

import numpy as np
import torch

from warp_drive_b200 import lib as _lib
from warp_drive_b200.utils.constants import Constants

_OBSERVATIONS = Constants.OBSERVATIONS
_ACTIONS = Constants.ACTIONS
_REWARDS = Constants.REWARDS
_DONE_FLAGS = Constants.DONE_FLAGS
_PROCESSED_OBSERVATIONS = Constants.PROCESSED_OBSERVATIONS


def _p(t):
    return _lib.ptr(t)


def fill_tc_env(dm, stats=None, with_scratch=False, write_observations=True):
    """wdb_tc_env from the arrays TagContinuous.get_data_dictionary registered."""
    env = _lib.TcEnv()
    env.n_envs = int(dm.meta_info("n_envs"))
    env.n_agents = int(dm.meta_info("n_agents"))
    for name in ("loc_x", "loc_y", "speed", "direction", "acceleration", "agent_types",
                 "edge_hit_reward_penalty", "acceleration_actions", "turn_actions",
                 "skill_levels", "still_in_the_game", "nearest_neighbor_ids", "step_rewards",
                 "num_runners"):
        setattr(env, name, _p(dm.device_data(name)))
    for name in ("edge_hit_penalty", "grid_length", "max_speed", "distance_margin_for_reward",
                 "tag_reward_for_tagger", "tag_penalty_for_runner",
                 "end_of_game_reward_for_runner"):
        setattr(env, name, float(dm.device_data(name)))
    for name in ("num_other_agents_observed", "runner_exits_game_after_tagged",
                 "use_full_observation"):
        setattr(env, name, int(dm.device_data(name)))
    env.obs = _p(dm.device_data(_OBSERVATIONS)) if write_observations else None
    env.rewards = _p(dm.device_data(_REWARDS))
    env.done = _p(dm.device_data("_done_"))
    env.env_timestep = _p(dm.device_data("_timestep_"))
    env.episode_length = int(dm.meta_info("episode_length"))
    env.stats = _p(stats)
    env.blocks_per_env = int(dm.meta_info("blocks_per_env"))
    if with_scratch and len(dm.get_shape("neighbor_distances")) == 3:
        env.neighbor_distances = _p(dm.device_data("neighbor_distances"))
        env.neighbor_ids_sorted_by_distance = _p(
            dm.device_data("neighbor_ids_sorted_by_distance"))
    return env


class FusedTagContinuousStep:
    @staticmethod
    def eligible(env_wrapper, policy_map, obs_tiles=False, actions_in=False):
        """Whether the library runs the fused step for this env, these policies, (with
        obs_tiles) the bf16 observation tiles and (with actions_in) actions sampled by the
        forward; it applies the same launch plan as the step."""
        ro = _lib.TcRollout()
        ro.actions_in = int(bool(actions_in))
        ro.n_policies = len(policy_map)
        heads = env_wrapper.env.action_space[0].nvec
        ro.n_actions0, ro.n_actions1 = int(heads[0]), int(heads[1])
        for pi, ids in enumerate(policy_map.values()):
            ro.policy[pi].n_agents = len(ids)
        env = fill_tc_env(env_wrapper.cuda_data_manager)
        return _lib.load().wdb_tag_continuous_rollout_supported(
            ctypes.byref(env), ctypes.byref(ro), int(bool(obs_tiles))) == 0

    def __init__(self, env_wrapper, policy_map, sampler, resetter=None, stats=None,
                 write_observations=True, write_head_actions=True):
        self.dm = dm = env_wrapper.cuda_data_manager
        self.device = dm.device
        self.E = env_wrapper.n_envs
        self.N = env_wrapper.n_agents
        self.policies = list(policy_map.keys())
        assert 1 <= len(self.policies) <= 4
        self.sampler = sampler
        self.lib = _lib.load()
        self.env = fill_tc_env(dm, stats=stats, write_observations=write_observations)
        ro = self.ro = _lib.TcRollout()
        ro.rng_state = _p(sampler.rng_state)
        ro.n_policies = len(self.policies)
        heads = env_wrapper.env.action_space[0].nvec
        ro.n_actions0, ro.n_actions1 = int(heads[0]), int(heads[1])
        agent_policy = np.zeros(self.N, np.int32)
        agent_slot = np.zeros(self.N, np.int32)
        for pi, p in enumerate(self.policies):
            for slot, a in enumerate(policy_map[p]):
                agent_policy[a], agent_slot[a] = pi, slot
        self._agent_policy = torch.from_numpy(agent_policy).to(self.device)
        self._agent_slot = torch.from_numpy(agent_slot).to(self.device)
        ro.agent_policy, ro.agent_slot = _p(self._agent_policy), _p(self._agent_slot)
        for pi, p in enumerate(self.policies):
            ro.policy[pi].n_agents = len(policy_map[p])
        ro.sampled_actions = _p(dm.device_data(_ACTIONS))
        if write_head_actions and dm.is_data_on_device(f"{_ACTIONS}_0"):
            ro.sampled_actions_0 = _p(dm.device_data(f"{_ACTIONS}_0"))
            ro.sampled_actions_1 = _p(dm.device_data(f"{_ACTIONS}_1"))
        if resetter is None:
            resetter = env_wrapper.env_resetter
        table, n = resetter.build_table(dm)
        assert not dm.reset_target_to_pool, "fused TagContinuous step has no pool reset"
        self._table = table
        ro.reset_table, ro.n_reset_arrays = _p(table), n
        ro.obs_at_reset = _p(dm.device_data(f"{_OBSERVATIONS}_at_reset"))
        ro.reset_done_envs = 1
        self._env_ref = ctypes.byref(self.env)
        self._ro_ref = ctypes.byref(self.ro)

    def set_bookkeeping(self, reward_running_sum, episodic_reward_sum, step_running_sum,
                        episodic_step_sum, num_completed):
        for pi, p in enumerate(self.policies):
            self.ro.policy[pi].reward_running_sum = _p(reward_running_sum[p])
            self.ro.policy[pi].episodic_reward_sum = _p(episodic_reward_sum[p])
        self.ro.step_running_sum = _p(step_running_sum)
        self.ro.episodic_step_sum = _p(episodic_step_sum)
        self.ro.num_completed_episodes = _p(num_completed)

    def launch(self, probs, actions_batch=None, rewards_batch=None, obs_next=None,
               done_batch=None, uniforms=None, reset_done_envs=True, obs_next_tiles=None,
               after_forward=False, actions_in=False, envs=None):
        """probs: {policy: [probs_head0 [E,Np,A0], probs_head1 [E,Np,A1]]}; the *_batch /
        obs_next dicts hold this timestep's slots (tensors) per policy, or None.
        actions_in: the forward already sampled the actions into `actions_batch` (required),
        which the step then reads instead of sampling from `probs` (may be None).
        envs: (begin, end), step only these envs (every tensor still covers all E)."""
        ro = self.ro
        for pi, p in enumerate(self.policies):
            io = ro.policy[pi]
            io.probs0, io.probs1 = (_p(probs[p][0]), _p(probs[p][1])) if probs else (None, None)
            io.actions_batch = _p(actions_batch[p]) if actions_batch else None
            io.rewards_batch = _p(rewards_batch[p]) if rewards_batch else None
            io.obs_next = _p(obs_next[p]) if obs_next else None
            io.obs_next_tiles = _p(obs_next_tiles[p]) if obs_next_tiles else None
        ro.done_batch = _p(done_batch)
        ro.uniforms = _p(uniforms)
        ro.reset_done_envs = int(bool(reset_done_envs))
        ro.launch_after_forward = int(bool(after_forward))
        ro.actions_in = int(bool(actions_in))
        ro.env_begin, ro.env_count = (0, 0) if envs is None else (envs[0], envs[1] - envs[0])
        _lib.check(self.lib.wdb_tag_continuous_rollout_step(
            _lib.stream_ptr(), self._env_ref, self._ro_ref), "tag_continuous_rollout_step")
