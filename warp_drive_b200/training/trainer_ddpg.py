"""TrainerDDPG: off-policy actor-critic training for continuous (Box) action spaces --
Pendulum and ContinuousMountainCar (SURVEY section 8 row f2).

Public surface of the reference's TrainerDDPG (warp_drive/training/trainers/
trainer_ddpg.py:52-532): same constructor, same run-config schema (`algorithm: "DDPG"`,
`tau`, `n_step`, per-network `lr.{actor,critic}` / `model.{actor,critic}`, `sampler.params`
for the OU noise), same `{policy}_actor_{t}.state_dict` / `{policy}_critic_{t}.state_dict`
checkpoints, same losses (algorithms/ddpg.py).

Underneath:
  * the rollout is ONE launch of the whole-rollout kernel (wdb_single_agent_rollout: actor
    forward -> Ornstein-Uhlenbeck exploration noise -> env step -> bookkeeping -> done-masked
    reset, incl. reset pools) for actors it supports (<= 3 hidden layers of width <= 64), else
    the device-resident generic step of RolloutEngine: actor forward ->
    wdb_sample_ou_process -> env step kernel -> bookkeeping -> reset; no host sync either way;
  * the replay window is the batch arrays themselves used as ONE ring (capacity
    `train_batch_size_per_env + n_step - 1`, trainer_base.py:246) with a single shared
    cursor -- every array is written in lock step, so the per-array queue objects of the
    reference (ring_buffer.py) collapse to two integers; `RingBuffer` is still provided
    for API parity (training/utils/ring_buffer.py);
  * the update is two launches per policy (wdb_ddpg_update, algorithms/fused_ddpg.py: every
    actor and critic gradient read in place from the ring) for the shapes it supports, else
    torch autograd over the unrolled ring;
  * one flat parameter / gradient arena over the actor and critic of every policy, with one
    FlatAdam (clipping + Adam as flat kernels) per network, so each network is clipped by its
    own norm as clip_grad_norm_ does; target networks are tracked with fused `torch._foreach`
    updates;
  * multi-GPU: one flat NCCL all-reduce over actor + critic gradients per iteration.

Replay buffer (trainer key `replay_slots_per_env`, see `replay_settings`): the same ring made
that many timesteps long, and `updates_per_iteration` updates after each rollout, each over
`replay_batch_rows` uniformly sampled n-step windows (wdb_replay_sample_windows) that the
*_sampled passes read in place.  The buffer is per GPU (each rank samples its own store with
its own seed) and is not checkpointed.
"""
import math
import os

import torch

from warp_drive_b200 import lib as _lib
from warp_drive_b200.training.algorithms.ddpg import DDPG
from warp_drive_b200.training.algorithms.fused_ddpg import FusedDDPGUpdate, fused_ddpg_supported
from warp_drive_b200.training.models.fully_connected_actor_critic import ActorAsPolicy
from warp_drive_b200.training.rollout import RolloutEngine
from warp_drive_b200.training.trainer import Trainer
from warp_drive_b200.training.utils.param_scheduler import ParamScheduler
from warp_drive_b200.utils.constants import Constants

_ACTIONS = Constants.ACTIONS
_REWARDS = Constants.REWARDS
_DONE_FLAGS = Constants.DONE_FLAGS
_PROCESSED_OBSERVATIONS = Constants.PROCESSED_OBSERVATIONS


def soft_update(target, source, tau):
    """target <- (1 - tau) * target + tau * source (trainer_ddpg.py:40-44), two fused launches."""
    tp, sp = list(target.parameters()), list(source.parameters())
    with torch.no_grad():
        torch._foreach_mul_(tp, 1.0 - tau)
        torch._foreach_add_(tp, sp, alpha=tau)


def hard_update(target, source):
    target.load_state_dict(source.state_dict())


_REPLAY_KEYS = ("replay_batch_rows", "updates_per_iteration", "replay_warmup_slots")


def replay_settings(trainer_config, batch_slots, n_step):
    """The validated replay-buffer keys of a trainer config, or None without
    `replay_slots_per_env` (the ring of one rollout, updated over every window).  Returns
    {"slots", "batch_rows" (None: one rollout's rows of the policy), "updates", "warmup"}."""
    slots = trainer_config.get("replay_slots_per_env")
    if slots is None:
        for key in _REPLAY_KEYS:
            if trainer_config.get(key) is not None:
                raise ValueError(f"{key} needs replay_slots_per_env")
        return None
    if int(slots) != slots or slots < batch_slots + n_step:
        raise ValueError(f"replay_slots_per_env must be an integer >= train_batch_size / "
                         f"num_envs + n_step = {batch_slots + n_step}, got {slots}")
    rows = trainer_config.get("replay_batch_rows")
    if rows is not None and (int(rows) != rows or not 1 <= rows < 2 ** 31):
        raise ValueError(f"replay_batch_rows must be an integer in [1, 2^31), got {rows}")
    updates = trainer_config.get("updates_per_iteration", 1)
    if int(updates) != updates or updates < 1:
        raise ValueError(f"updates_per_iteration must be an integer >= 1, got {updates}")
    warmup = trainer_config.get("replay_warmup_slots", batch_slots + n_step)
    if int(warmup) != warmup or not n_step + 1 <= warmup <= slots:
        raise ValueError(f"replay_warmup_slots must be an integer in [n_step + 1, "
                         f"replay_slots_per_env] = [{n_step + 1}, {slots}], got {warmup}")
    return {"slots": int(slots), "batch_rows": None if rows is None else int(rows),
            "updates": int(updates), "warmup": int(warmup)}


_PRIORITY_KEYS = ("priority_alpha", "priority_beta", "priority_epsilon")


def _unit_number(v):
    return isinstance(v, (int, float)) and not isinstance(v, bool) and 0 <= v <= 1


def prioritized_settings(trainer_config, replay):
    """The validated prioritized-replay keys of a trainer config, or None without
    `prioritized_replay`.  `replay`: replay_settings' result.  Returns {"alpha", "beta" (a
    ParamScheduler over the policy timestep), "epsilon"}."""
    if not trainer_config.get("prioritized_replay"):
        for key in _PRIORITY_KEYS:
            if trainer_config.get(key) is not None:
                raise ValueError(f"{key} needs prioritized_replay")
        return None
    if trainer_config["prioritized_replay"] is not True:
        raise ValueError(f"prioritized_replay is True or False, got "
                         f"{trainer_config['prioritized_replay']!r}")
    if replay is None:
        raise ValueError("prioritized_replay needs replay_slots_per_env")
    alpha = trainer_config.get("priority_alpha", 0.6)
    if not _unit_number(alpha):
        raise ValueError(f"priority_alpha must lie in [0, 1], got {alpha}")
    beta = trainer_config.get("priority_beta", 0.5)
    knots = beta if isinstance(beta, list) else [[0, beta]]
    if not knots or not all(isinstance(k, (list, tuple)) and len(k) == 2 and _unit_number(k[1])
                            for k in knots):
        raise ValueError(f"priority_beta must be a number or [[t, v], ...] with v in [0, 1], "
                         f"got {beta}")
    if [k[0] for k in knots] != sorted(k[0] for k in knots):
        raise ValueError(f"priority_beta's timesteps must be increasing, got {beta}")
    eps = trainer_config.get("priority_epsilon", 1e-6)
    if not (isinstance(eps, (int, float)) and not isinstance(eps, bool) and 0 < eps
            and math.isfinite(eps)):
        raise ValueError(f"priority_epsilon must be a finite number > 0, got {eps}")
    return {"alpha": float(alpha), "beta": ParamScheduler(beta), "epsilon": float(eps)}


class RingRolloutEngine(RolloutEngine):
    """RolloutEngine whose batch index wraps: timestep t of a rollout lands in slot
    (cursor + t) mod capacity of every `*_batch*` array."""

    def __init__(self, *args, ring_capacity=None, **kwargs):
        kwargs.update(use_cuda_graph=False)
        super().__init__(*args, **kwargs)
        assert ring_capacity is not None and ring_capacity >= self.T
        self.ring_capacity = int(ring_capacity)
        self.ring_cursor = 0          # slot of the next timestep
        self.ring_filled = 0          # valid slots (<= capacity)

    def _fused_eligible(self):
        # the tag_continuous per-step kernel writes batch slot t itself (no ring mapping)
        return False

    def _slot(self, t):
        return t if t < 0 else (self.ring_cursor + t) % self.ring_capacity

    def rollout(self, **sample_params):
        if self.sa is not None and self._sa_params_ok(sample_params):
            # slots cursor .. cursor + T - 1 (mod capacity): at most two launches, split at
            # the wrap point
            with torch.no_grad():
                first = min(self.T, self.ring_capacity - self.ring_cursor)
                self.sa.launch(first, t0=self.ring_cursor, **sample_params)
                if first < self.T:
                    self.sa.launch(self.T - first, t0=0, **sample_params)
        else:
            self._rollout_eager(**sample_params)
        self.ring_cursor = (self.ring_cursor + self.T) % self.ring_capacity
        self.ring_filled = min(self.ring_capacity, self.ring_filled + self.T)

    def isfull(self):
        return self.ring_filled == self.ring_capacity

    def unroll(self, name):
        """Time-ordered contents (oldest first) of batch array `name`."""
        q = self._tensor(name)
        if self.ring_filled < self.ring_capacity:
            return q[:self.ring_filled]
        if self.ring_cursor == 0:
            return q
        return torch.cat((q[self.ring_cursor:], q[:self.ring_cursor]), dim=0)


class TrainerDDPG(Trainer):
    """Trainer's setup, update tail and checkpointing; what differs is an actor, a critic and
    their target networks per policy, the replay ring and the DDPG update."""

    def __init__(self, env_wrapper=None, config=None, policy_tag_to_agent_id_map=None,
                 create_separate_placeholders_for_each_policy=False,
                 obs_dim_corresponding_to_num_agents="first", num_devices=1, device_id=0,
                 results_dir=None, verbose=True):
        assert not create_separate_placeholders_for_each_policy, (
            "TrainerDDPG steps every policy through the shared observation / action / reward "
            "arrays: separate per-policy placeholders are not supported")
        if config is not None:
            from warp_drive_b200.training.obs_norm import refuse_obs_norm
            from warp_drive_b200.training.reward_scale import refuse_reward_scale

            refuse_obs_norm(config, type(self).__name__)
            refuse_reward_scale(config, type(self).__name__)
        super().__init__(env_wrapper, config, policy_tag_to_agent_id_map,
                         create_separate_placeholders_for_each_policy,
                         obs_dim_corresponding_to_num_agents, num_devices, device_id,
                         results_dir, verbose, use_cuda_graph=False)

    # the trainer key prioritized_replay (TrainerDQN); the actor-critic passes have no weights
    _takes_prioritized_replay = False

    # ------------------------------------------------------------------ setup
    @staticmethod
    def _check_obs_dim(obs_dim_corresponding_to_num_agents):
        """Either layout is passed on to the step placeholders as given."""

    @staticmethod
    def _merge_policy_defaults(policy_config, defaults):
        # actor / critic sub-dicts of `model` and `lr` are kept as given
        for k, v in defaults.items():
            policy_config.setdefault(k, v)

    def _batch_slots_per_env(self, trainer_config):
        """The replay ring: one rollout plus the n_step - 1 slots the n-step target looks
        ahead."""
        self.n_step = int(trainer_config.get("n_step", 1))
        assert self.n_step >= 1
        self.replay = replay_settings(trainer_config, self.training_batch_size_per_env,
                                      self.n_step)
        self.prioritized = prioritized_settings(trainer_config, self.replay)
        if self.prioritized is not None and not self._takes_prioritized_replay:
            raise ValueError(f"prioritized_replay is DQN's: {type(self).__name__} samples its "
                             f"replay windows uniformly")
        if self.replay is not None:
            self.ring_capacity = self.replay["slots"]
        else:
            self.ring_capacity = self.training_batch_size_per_env + self.n_step - 1
        return self.ring_capacity

    def _create_network_dicts(self):
        self.actor_models, self.critic_models = {}, {}
        self.target_actor_models, self.target_critic_models = {}, {}
        self.actor_optimizers, self.critic_optimizers = {}, {}
        self.actor_lr_schedules, self.critic_lr_schedules = {}, {}
        self.tau, self.fused_updates = {}, {}
        self.replay_windows, self.replay_draws = {}, 0
        # `models`: the networks the rollout runs
        self.models = self.actor_models

    def _split(self, policy, key):
        """(actor part, critic part) of a config entry that may or may not be split."""
        value = self._get_config(["policy", policy, key])
        if isinstance(value, dict) and "actor" in value and "critic" in value:
            return value["actor"], value["critic"]
        return value, value

    def _initialize_policy_model(self, policy):
        actor_cfg, critic_cfg = self._split(policy, "model")
        self.actor_models[policy] = self._build_model(policy, actor_cfg)
        self.target_actor_models[policy] = self._build_model(policy, actor_cfg)
        hard_update(self.target_actor_models[policy], self.actor_models[policy])
        self.critic_models[policy] = self._build_model(policy, critic_cfg)
        self.target_critic_models[policy] = self._build_model(policy, critic_cfg)
        hard_update(self.target_critic_models[policy], self.critic_models[policy])

    def _trained_networks(self, policy):
        return [self.actor_models[policy], self.critic_models[policy]]

    def _all_networks(self, policy):
        return self._trained_networks(policy) + [self.target_actor_models[policy],
                                                 self.target_critic_models[policy]]

    def _initialize_optimizer(self, policy):
        actor_lr, critic_lr = self._split(policy, "lr")
        self.actor_lr_schedules[policy] = ParamScheduler(actor_lr)
        self.critic_lr_schedules[policy] = ParamScheduler(critic_lr)
        ts = self.current_timestep[policy]
        self.actor_optimizers[policy] = self._flat_adam(
            self.actor_models[policy], self.actor_lr_schedules[policy].get_param_value(ts))
        self.critic_optimizers[policy] = self._flat_adam(
            self._critic_optimized(policy), self.critic_lr_schedules[policy].get_param_value(ts))

    def _critic_optimized(self, policy):
        """The module whose parameters the critic's optimizer steps (and clips together)."""
        return self.critic_models[policy]

    def _optimizers_of(self, policy):
        return [(" (Actor)", self.actor_optimizers[policy], self.actor_lr_schedules[policy]),
                (" (Critic)", self.critic_optimizers[policy], self.critic_lr_schedules[policy])]

    def _initialize_policy_algorithm(self, policy):
        c = self._get_config(["policy", policy])
        assert c["algorithm"] == "DDPG"
        self.clip_grad_norm[policy] = c["clip_grad_norm"]
        if c["clip_grad_norm"]:
            self.max_grad_norm[policy] = c["max_grad_norm"]
        self.tau[policy] = c["tau"]
        self.trainers[policy] = DDPG(
            discount_factor_gamma=c["gamma"], normalize_advantage=c["normalize_advantage"],
            normalize_return=c["normalize_return"], n_step=self.n_step)
        n_agents = len(self.policy_tag_to_agent_id_map[policy])
        args = (self.num_envs, n_agents, self.ring_capacity, self.n_step)
        actor, critic = self.actor_models[policy], self.critic_models[policy]
        rows = self._init_replay(policy)
        if fused_ddpg_supported(self.trainers[policy], actor, critic, *args, replay_rows=rows):
            self.fused_updates[policy] = FusedDDPGUpdate(
                actor, critic, self.target_actor_models[policy],
                self.target_critic_models[policy], *args, gamma=c["gamma"], replay_rows=rows)

    def _init_replay(self, policy):
        """With a replay buffer: the policy's window buffer (int32 [B, 2]) and the log line
        of the store's size.  Returns B, the loss rows per update (None without a buffer)."""
        if self.replay is None:
            return None
        n_agents = len(self.policy_tag_to_agent_id_map[policy])
        rows = self.replay["batch_rows"]
        if rows is None:
            rows = self.training_batch_size_per_env * self.num_envs * n_agents
        dev = next(self.actor_models[policy].parameters()).device
        self.replay_windows[policy] = torch.zeros((rows, 2), dtype=torch.int32, device=dev)
        dm = self.cuda_envs.cuda_data_manager
        names = [f"{_PROCESSED_OBSERVATIONS}_batch_{policy}", f"{_ACTIONS}_batch_{policy}",
                 f"{_REWARDS}_batch_{policy}", f"{_DONE_FLAGS}_batch"]
        nbytes = sum(t.numel() * t.element_size()
                     for t in map(dm.data_on_device_via_torch, names))
        if self.verbose:
            print(f"[Device {self.device_id}]: replay buffer of policy '{policy}': "
                  f"{self.ring_capacity} slots x {self.num_envs} envs x {n_agents} agents = "
                  f"{self.ring_capacity * self.num_envs * n_agents} transitions, {nbytes} "
                  f"bytes on the device; {rows} rows per update, {self.replay['updates']} "
                  f"updates per iteration")
        return rows

    def _make_engine(self, use_cuda_graph):
        engine = RingRolloutEngine(
            self.cuda_envs, {p: ActorAsPolicy(self.actor_models[p]) for p in self.policies},
            self.policy_tag_to_agent_id_map, self.cuda_sample_controller,
            self.training_batch_size_per_env, ring_capacity=self.ring_capacity)
        assert engine.continuous, "DDPG needs a continuous (Box) action space"
        return engine

    # ------------------------------------------------------------------ update
    def _update_model_params(self, iteration):
        """After a rollout: nothing while the ring fills; then one update over every window of
        the ring, or -- with a replay buffer -- `updates_per_iteration` updates over freshly
        sampled windows.  Only the last update of a logging iteration collects metrics."""
        logging_flag = self._is_logging_iteration(iteration)
        loss_metrics = {}
        step_info = {policy: ({}, {}) for policy in self.policies_to_train}
        if self._ready_to_update():
            for policy in self.policies_to_train:
                self._advance_timestep(policy)
            updates = 1 if self.replay is None else self.replay["updates"]
            for k in range(updates):
                loss_metrics = self._one_update(logging_flag and k == updates - 1, step_info)
        metrics_dict = self._finish_update(loss_metrics, step_info, logging_flag)
        if self.replay is not None:
            for metrics in metrics_dict.values():
                metrics["Replay buffer fill"] = self.engine.ring_filled / self.ring_capacity
        self._add_test_metrics(metrics_dict, logging_flag)
        return metrics_dict

    def _ready_to_update(self):
        """Until then the rollouts only fill the ring."""
        if self.replay is None:
            return self.engine.isfull()
        return self.engine.ring_filled >= self.replay["warmup"]

    def _one_update(self, logging_flag, step_info):
        """Gradients, optimizer steps and target tracking of every trained policy; returns
        their loss metrics (filled when logging_flag)."""
        loss_metrics = {}
        for policy in self.policies_to_train:
            self._sample_replay_windows(policy)
            fused = self.fused_updates.get(policy)
            if fused is not None and self.trainers[policy].use_fused_update:
                loss_metrics[policy] = self._fused_gradients(policy, fused, logging_flag)
            elif self.replay is not None:
                loss_metrics[policy] = self._torch_replay_gradients(policy, logging_flag)
            else:
                loss_metrics[policy] = self._torch_gradients(policy, logging_flag)
        step_info.update(self._optimizer_step(loss_metrics, logging_flag))
        for policy in loss_metrics:
            soft_update(self.target_actor_models[policy], self.actor_models[policy],
                        self.tau[policy])
            soft_update(self.target_critic_models[policy], self.critic_models[policy],
                        self.tau[policy])
        return loss_metrics

    # ------------------------------------------------------------------ replay buffer
    def _sample_replay_windows(self, policy):
        """With a replay buffer: draws this update's windows of `policy` on the device into
        replay_windows[policy] (one launch, no host wait).  The draw is a function of the
        trainer seed (rank-dependent) and the running draw count."""
        if self.replay is None:
            return
        eng, windows = self.engine, self.replay_windows[policy]
        self.replay_draws += 1
        oldest = eng.ring_cursor if eng.ring_filled == eng.ring_capacity else 0
        n_agents = len(self.policy_tag_to_agent_id_map[policy])
        _lib.check(_lib.load().wdb_replay_sample_windows(
            _lib.stream_ptr(), _lib.ptr(windows), int(windows.shape[0]), self.seed,
            self.replay_draws, oldest, eng.ring_filled, eng.ring_capacity, self.n_step,
            self.num_envs * n_agents), "replay_sample_windows")

    def _gather_windows(self, policy):
        """The sampled windows of `policy` gathered by index from the physical ring (never
        unrolled: that would copy all of it): obs [B, F], actions [B, A], rewards [n_step, B],
        done [n_step, B] (float), bootstrap obs [B, F]."""
        eng, C = self.engine, self.ring_capacity
        windows = self.replay_windows[policy].long()
        start, row = windows[:, 0], windows[:, 1]
        steps = (start[None, :] + torch.arange(self.n_step + 1, device=start.device)[:, None]) % C
        obs = eng._tensor(f"{_PROCESSED_OBSERVATIONS}_batch_{policy}")
        actions = eng._tensor(f"{_ACTIONS}_batch_{policy}")
        rewards = eng._tensor(f"{_REWARDS}_batch_{policy}")
        done = eng._tensor(f"{_DONE_FLAGS}_batch")
        n_agents = rewards.shape[2]
        obs = obs.reshape(C, -1, obs.shape[-1])
        return (obs[start, row], actions.reshape(C, -1, actions.shape[-1])[start, row],
                rewards.reshape(C, -1)[steps[:-1], row],
                done[steps[:-1], row // n_agents].to(rewards.dtype), obs[steps[-1], row])

    @staticmethod
    def _batch_metrics(metrics):
        """Metrics of a sampled batch (laid out as one timestep of B envs): the spreads over
        agents and over time do not exist for it and are dropped."""
        return {k: v for k, v in metrics.items() if not (isinstance(v, float) and math.isnan(v))}

    def _torch_replay_gradients(self, policy, logging_flag):
        """_torch_gradients over the sampled windows: the losses of wdb_ddpg_update_sampled by
        torch autograd on the gathered batch."""
        algo = self.trainers[policy]
        obs, actions, rewards, done, boot_obs = self._gather_windows(policy)
        actor, critic = self.actor_models[policy], self.critic_models[policy]
        with torch.no_grad():
            boot = self.target_critic_models[policy](
                obs=boot_obs, action=self.target_actor_models[policy](obs=boot_obs))
            returns = algo.sampled_returns(rewards, done, boot)
        values = critic(obs=obs, action=actions)
        j_values = critic(obs=obs, action=actor(obs=obs))
        actor_loss, critic_loss = -j_values.mean(), torch.nn.functional.mse_loss(values, returns)
        self.actor_optimizers[policy].zero_grad()
        self.critic_optimizers[policy].zero_grad()
        actor_loss.backward()
        critic_loss.backward()
        if not logging_flag:
            return {}
        return self._batch_metrics(algo.loss_metrics(
            actor_loss.item(), critic_loss.item(), rewards[0][None, :, None],
            actions[None, :, None], values.detach()[None, :, None],
            j_values.detach()[None, :, None], returns[None, :, None]))

    # the sampler arguments of the evaluator's noise-free test episodes
    _test_sample_params = {"scale": 0}

    def _add_test_metrics(self, metrics_dict, logging_flag):
        """On a logging iteration with the evaluator on: noise-free test episodes' metrics."""
        if logging_flag and self.config["trainer"].get("evaluator"):
            reward_sum, step_sum = self.evaluate_episodes(**self._test_sample_params)
            for policy in self.policies_to_train:
                metrics_dict[policy].update({
                    "Mean episodic reward (test)": float(reward_sum[policy].mean()),
                    "Mean episodic steps (test)": float(step_sum[policy].float().mean())})

    def _torch_gradients(self, policy, logging_flag):
        """Actor / critic gradients by torch autograd over the unrolled ring (accumulated into
        the arena's .grad views); returns the metrics of a logging iteration."""
        eng = self.engine
        done_flags = eng.unroll(f"{_DONE_FLAGS}_batch")
        actions = eng.unroll(f"{_ACTIONS}_batch_{policy}")
        rewards = eng.unroll(f"{_REWARDS}_batch_{policy}")
        obs = eng.unroll(f"{_PROCESSED_OBSERVATIONS}_batch_{policy}")
        actor, critic = self.actor_models[policy], self.critic_models[policy]
        probs = actor(obs=obs)
        with torch.no_grad():
            target_probs = self.target_actor_models[policy](obs=obs)
            next_values = self.target_critic_models[policy](
                obs=obs[1:], action=[p[1:] for p in target_probs])
        values = critic(obs=obs, action=actions)
        j_values = critic(obs=obs, action=probs)
        actor_loss, critic_loss, metrics = self.trainers[policy].compute_loss_and_metrics(
            self.current_timestep[policy], actions, rewards, done_flags, values,
            next_values, j_values, perform_logging=logging_flag)
        self.actor_optimizers[policy].zero_grad()
        self.critic_optimizers[policy].zero_grad()
        # the order and the (shared) critic gradient of the reference
        # (trainer_ddpg.py:412-415): the actor loss also back-propagates into the critic
        actor_loss.backward()
        critic_loss.backward()
        return metrics

    def _fused_gradients(self, policy, fused, logging_flag):
        """The same gradients as _torch_gradients from wdb_ddpg_update, written straight into
        the arena's .grad views; the host waits only on logging iterations (metrics)."""
        eng = self.engine
        rewards = eng._tensor(f"{_REWARDS}_batch_{policy}")
        actions = eng._tensor(f"{_ACTIONS}_batch_{policy}")
        windows = self.replay_windows.get(policy)
        outputs = None
        if logging_flag:
            shape = (fused.valid,) + tuple(rewards.shape[1:]) if windows is None else (
                1, fused.rows, 1)
            outputs = tuple(torch.empty(shape, device=rewards.device) for _ in range(3))
        sums = fused.launch(eng._tensor(f"{_PROCESSED_OBSERVATIONS}_batch_{policy}"), actions,
                            rewards, eng._tensor(f"{_DONE_FLAGS}_batch"), eng.ring_cursor,
                            outputs, windows=windows)
        if not logging_flag:
            return {}
        s = sums.tolist()
        values, j_values, returns = outputs
        if windows is not None:       # the metrics of the sampled rows' first step
            _, actions, rewards, _, _ = self._gather_windows(policy)
            return self._batch_metrics(self.trainers[policy].loss_metrics(
                -s[1] / fused.rows, s[0] / fused.rows, rewards[0][None, :, None],
                actions[None, :, None], values, j_values, returns))
        # the ring in slot order: the metrics are means / extremes / spreads over all of it
        return self.trainers[policy].loss_metrics(
            -s[1] / fused.rows, s[0] / fused.rows, rewards, actions, values, j_values, returns)

    # ------------------------------------------------------------------ checkpoints
    def _checkpointed_networks(self):
        return [(policy, f"{policy}_{kind}", model)
                for kind, models in (("actor", self.actor_models), ("critic", self.critic_models))
                for policy, model in models.items()]

    def _load_policy_checkpoint(self, policy, paths):
        if not (isinstance(paths, dict) and paths.get("actor") and paths.get("critic")):
            return
        assert os.path.isfile(paths["actor"]), "Invalid actor model checkpoint path!"
        assert os.path.isfile(paths["critic"]), "Invalid critic model checkpoint path!"
        steps = [self._checkpoint_timestep(paths[k]) for k in ("actor", "critic")]
        assert steps[0] == steps[1], (
            "The timestep is different between the actor model and the critic model ")
        self.actor_models[policy].load_state_dict(torch.load(paths["actor"], map_location="cpu"))
        self.critic_models[policy].load_state_dict(torch.load(paths["critic"], map_location="cpu"))
        hard_update(self.target_actor_models[policy], self.actor_models[policy])
        hard_update(self.target_critic_models[policy], self.critic_models[policy])
        self.current_timestep[policy] = steps[0]
