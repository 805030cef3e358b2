"""TrainerDQN: double DQN with n-step returns and a Huber loss (algorithms/dqn.py) for envs
with one Discrete action -- a policy with `algorithm: "DQN"` in its run config.

TrainerDDPG's replay buffer (`replay_slots_per_env` is required: DQN always trains from it),
window drawing, gradient arena, optimizer step, evaluator and checkpoint plumbing; what
differs is one Q network (`fully_connected_q`) and its target per policy:

  * the rollout samples actions epsilon-greedily from the Q network's raw outputs
    (CUDASampler.sample_epsilon_greedy on the engine's per-step path), with epsilon the one
    sampler param, a ParamScheduler schedule over the policy timestep;
  * per update: the windows (1 launch), the Q gradient (wdb_dqn_update_sampled, 2 launches, or
    torch autograd on the gathered windows for the shapes it does not take), the all-reduce,
    clipping + Adam (2 launches), and on every `target_update_period`-th update the target
    tracking with `tau` (1: a copy);
  * checkpoints `{policy}_q_{t}.state_dict`; `model_ckpt_filepath` is one path, and the target
    is a copy of the loaded network.

Policy keys: `double_q` (True), `huber_delta` (1.0), `tau` (1.0), `target_update_period` (1),
and Trainer's `lr`, `model`, `gamma`, `clip_grad_norm`, `max_grad_norm`; trainer key `n_step`.

Prioritized replay (trainer key `prioritized_replay`, see trainer_ddpg.prioritized_settings):
each policy's windows carry priorities in a device sum tree (utils/prioritized_replay.py).  Every
rollout admits its windows at the running maximum priority (wdb_per_admit), each update draws
its windows by stratified proportional sampling with importance-sampling weights
(wdb_per_sample_windows, beta from `priority_beta` over the policy timestep), takes the weighted
gradient (wdb_dqn_update_prioritized, or the weighted torch loss) and writes the windows' new
priorities (wdb_per_set_priorities) before the optimizer step.

Quantile-regression DQN: a `fully_connected_quantile_q` model (`num_quantiles` N) trains with
QuantileDQN's quantile Huber loss (wdb_qr_dqn_update_sampled, 2 launches, or torch autograd)
on the same windows, targets and schedule.  Its `Mean Q value` and `Mean return` are the means
of Q-bar = mean_i theta_i and R-bar = mean_j T_j, and with prioritized replay the priorities are
(|Q-bar - R-bar| + epsilon)^alpha.

Implicit quantile networks: a `fully_connected_iqn` model trains with ImplicitQuantileDQN's
quantile Huber loss over sampled levels (wdb_iqn_update_sampled, 2 launches, or torch autograd)
on the same windows, targets and schedule.  Each update draws its levels -- N online and N'
target ones per loss row, uniform on [0, 1) -- into one [B, N + N'] buffer with a CUDA
generator seeded from the trainer seed (1 launch); the native and the torch path read the same
buffer.  Metrics and priorities are QR-DQN's.

Categorical DQN (C51): a `fully_connected_categorical_q` model (`num_atoms` N, `v_min`, `v_max`)
trains with CategoricalDQN's projected cross-entropy (wdb_c51_update_sampled, 2 launches, or
torch autograd) on the same windows, targets and schedule.  C51 has no Huber loss, so a
categorical policy config that sets `huber_delta` is refused.  Its `Mean Q value` and `Mean
return` are the means of Q-bar = sum_i z_i p_i and R-bar = sum_i z_i m_i, and with prioritized
replay the priorities are (|Q-bar - R-bar| + epsilon)^alpha, as for QR-DQN and IQN (Rainbow
uses the cross-entropy).

Dueling: a `fully_connected_q` or `fully_connected_categorical_q` model with `dueling: true`
(and `stream_fc_dims` [] or [S]) trains with the same losses, windows, targets and schedule.
Per update the native path folds the online and target heads (wdb_dueling_fold, 1 launch), runs
the plain pass on the folded network (2 launches) and unfolds its head gradients onto the two
streams (wdb_dueling_unfold_grads, 1 launch); shapes outside the pass's envelope train through
torch autograd on the DuelingHead.

Noisy networks: a `fully_connected_q` or `fully_connected_categorical_q` model with `noisy: true`
(plain or dueling) explores through factorized Gaussian noise on its head.  Per update the native
path (FusedNoisyUpdate) draws one sample for the online head and an independent one for the
target, keyed by the trainer seed and the policy's update count, and writes the effective layers
(wdb_noisy_materialize, 1 launch), runs the plain or dueling pass on them, and maps their
gradients onto mu and sigma (wdb_noisy_grads, 1 launch); the online sample serves obs and obs'
alike, the double-Q argmax included.  The torch path draws the same sample into the layers' noise
buffers (wdb_noisy_draw) and differentiates through NoisyLinear.materialized().  Acting draws
fresh noise per env row and step on the rollout engine's per-step path; the evaluator plays the
mean network.  Logging iterations add `Noisy sigma`, the mean |sigma_W| over the head's noisy
layers.

Action masks: a Q model with `masked: true` over a Dict observation with an `action_mask` key
acts epsilon-greedily over the valid actions of each step's mask
(CUDASampler.sample_epsilon_greedy with `action_mask`), and the evaluator plays the masked greedy action.  The ring stores each
step's mask in action_mask_batch_{p}, and every update bootstraps over the valid actions of
obs' own mask, the row at the window's slot(n_step): the native DQN and C51 passes, plain,
dueling or noisy, through wdb_dqn_update_masked / wdb_c51_update_masked (FusedMaskedDQNUpdate,
FusedMaskedC51Update), and QR-DQN, IQN and every shape outside the passes through the torch
losses' `boot_mask`.  A row with no valid action falls back to the unmasked rule.

Action branching: a `fully_connected_branching_q` model over a MultiDiscrete action space
(Tavakoli, Pardo & Kormushev 2018) has one Q head per action dimension on a shared trunk.  The
rollout samples each head epsilon-greedily on its own (CUDASampler.sample_epsilon_greedy with
`branch_sizes`, one launch), the ring keeps the D actions of every step, and BranchingDQN's loss
regresses every head on the return built from the mean of the heads' bootstraps
(wdb_branching_dqn_update_sampled / _prioritized, 2 launches, or torch autograd).  `Mean Q value`
is the mean of Q-bar, the mean over the heads of Q_d(obs, a_d), and with prioritized replay the
priorities are (|Q-bar - R| + epsilon)^alpha.
"""
import os

import torch

from warp_drive_b200.training.algorithms.dqn import (
    DQN, BranchingDQN, CategoricalDQN, ImplicitQuantileDQN, QuantileDQN)
from warp_drive_b200.training.algorithms.fused_dqn import (
    NOISY_UPDATE, FusedBranchingDQNUpdate, FusedC51Update, FusedDQNUpdate, FusedDuelingUpdate,
    FusedIQNUpdate,
    FusedMaskedC51Update, FusedMaskedDQNUpdate, FusedNoisyUpdate, FusedQRDQNUpdate, draw_noise)
from warp_drive_b200.training.trainer_ddpg import (
    RingRolloutEngine, TrainerDDPG, hard_update, soft_update)
from warp_drive_b200.training.utils.param_scheduler import ParamScheduler
from warp_drive_b200.training.utils.prioritized_replay import PrioritizedReplay
from warp_drive_b200.utils.constants import Constants

_ACTIONS = Constants.ACTIONS
_REWARDS = Constants.REWARDS
_DONE_FLAGS = Constants.DONE_FLAGS
_PROCESSED_OBSERVATIONS = Constants.PROCESSED_OBSERVATIONS
_ACTION_MASK = Constants.ACTION_MASK


def epsilon_schedule(config):
    """The validated `sampler.params.epsilon` of a DQN run config: a number or [[t, v], ...] in
    [0, 1], and no other sampler param."""
    params = dict(config.get("sampler", {}).get("params", {}) or {})
    if "epsilon" not in params:
        raise ValueError("DQN explores epsilon-greedily: set sampler.params.epsilon")
    others = sorted(k for k in params if k != "epsilon")
    if others:
        raise ValueError(f"DQN takes the sampler param epsilon only, got also {others}")
    eps = params["epsilon"]
    values = [v for _, v in eps] if isinstance(eps, list) else [eps]
    if not all(isinstance(v, (int, float)) and 0 <= v <= 1 for v in values):
        raise ValueError(f"epsilon must lie in [0, 1], got {eps}")
    return ParamScheduler(eps)


def dqn_policy_settings(policy_config):
    """(double_q, huber_delta, tau, target_update_period) of a DQN policy config, validated."""
    c = policy_config
    if c.get("normalize_return"):
        raise ValueError("DQN does not take normalize_return")
    delta = c.get("huber_delta", 1.0)
    if not delta > 0:
        raise ValueError(f"huber_delta must be > 0, got {delta}")
    tau = c.get("tau", 1.0)
    if not 0 < tau <= 1:
        raise ValueError(f"tau must lie in (0, 1], got {tau}")
    period = c.get("target_update_period", 1)
    if int(period) != period or period < 1:
        raise ValueError(f"target_update_period must be an integer >= 1, got {period}")
    return bool(c.get("double_q", True)), float(delta), float(tau), int(period)


def categorical_policy_settings(policy_config):
    """dqn_policy_settings of a policy with a categorical (C51) Q network, which has no Huber
    loss: a `huber_delta` set in its config is refused rather than ignored."""
    if "huber_delta" in policy_config:
        raise ValueError("a fully_connected_categorical_q policy has no Huber loss: remove "
                         f"huber_delta (got {policy_config['huber_delta']!r})")
    return dqn_policy_settings(policy_config)


class TrainerDQN(TrainerDDPG):
    """TrainerDDPG's setup, replay buffer and checkpointing with one Q network and its target
    per policy and the DQN update."""

    # the evaluator plays greedily
    _test_sample_params = {"epsilon": 0}
    _takes_prioritized_replay = True

    def __init__(self, env_wrapper=None, config=None, policy_tag_to_agent_id_map=None,
                 create_separate_placeholders_for_each_policy=False,
                 obs_dim_corresponding_to_num_agents="first", num_devices=1, device_id=0,
                 results_dir=None, verbose=True):
        if create_separate_placeholders_for_each_policy:
            raise ValueError("DQN steps every policy through the shared observation / action / "
                             "reward arrays: separate per-policy placeholders are not supported")
        epsilon_schedule(config)
        super().__init__(env_wrapper, config, policy_tag_to_agent_id_map, False,
                         obs_dim_corresponding_to_num_agents, num_devices, device_id,
                         results_dir, verbose)

    # ------------------------------------------------------------------ setup
    def _batch_slots_per_env(self, trainer_config):
        slots = super()._batch_slots_per_env(trainer_config)
        if self.replay is None:
            raise ValueError("DQN trains from a replay buffer: set the trainer key "
                             "replay_slots_per_env")
        return slots

    def _create_network_dicts(self):
        self.q_models, self.target_q_models = {}, {}
        self.optimizers, self.lr_schedules = {}, {}
        self.tau, self.target_update_period, self.update_count = {}, {}, {}
        self.fused_updates, self.replay_windows, self.replay_draws = {}, {}, 0
        self.priority_stores = {}
        # IQN: each policy's levels of one update [B, N + N'] and the generator that draws them
        self.iqn_taus, self._tau_generator = {}, None
        self.last_epsilon = None
        # the networks the rollout runs (TrainerDDPG's replay helpers know them as actors)
        self.models = self.actor_models = self.q_models

    def _initialize_policy_model(self, policy):
        c = self._get_config(["policy", policy])
        if c.get("algorithm") != "DQN":
            raise ValueError(f"TrainerDQN trains algorithm DQN, policy '{policy}' has "
                             f"'{c.get('algorithm')}'")
        model_cfg = c["model"]
        self.q_models[policy] = self._build_model(policy, model_cfg)
        if not getattr(self.q_models[policy], "is_q_network", False):
            raise ValueError("DQN's model is a `fully_connected_q`, a `fully_connected_quantile_q`, "
                             "a `fully_connected_iqn`, a `fully_connected_categorical_q` or a "
                             f"`fully_connected_branching_q`, got '{model_cfg.get('type')}'")
        self.target_q_models[policy] = self._build_model(policy, model_cfg)
        hard_update(self.target_q_models[policy], self.q_models[policy])

    def _trained_networks(self, policy):
        return [self.q_models[policy]]

    def _all_networks(self, policy):
        return [self.q_models[policy], self.target_q_models[policy]]

    def _initialize_optimizer(self, policy):
        self.lr_schedules[policy] = ParamScheduler(self._get_config(["policy", policy, "lr"]))
        self.optimizers[policy] = self._flat_adam(
            self.q_models[policy],
            self.lr_schedules[policy].get_param_value(self.current_timestep[policy]))

    def _optimizers_of(self, policy):
        return [("", self.optimizers[policy], self.lr_schedules[policy])]

    def _initialize_policy_algorithm(self, policy):
        c = self._get_config(["policy", policy])
        q_net = self.q_models[policy]
        categorical = getattr(q_net, "is_categorical_q", False)
        double_q, delta, tau, period = (
            categorical_policy_settings if categorical else dqn_policy_settings)(c)
        self.clip_grad_norm[policy] = c["clip_grad_norm"]
        if c["clip_grad_norm"]:
            self.max_grad_norm[policy] = c["max_grad_norm"]
        self.tau[policy], self.target_update_period[policy] = tau, period
        self.update_count[policy] = 0
        quantile = getattr(q_net, "is_quantile_q", False)
        implicit = getattr(q_net, "is_implicit_quantile_q", False)
        branching = getattr(q_net, "is_branching_q", False)
        algo = self.trainers[policy] = (
            CategoricalDQN if categorical else ImplicitQuantileDQN if implicit
            else QuantileDQN if quantile else BranchingDQN if branching else DQN)(
            discount_factor_gamma=c["gamma"], n_step=self.n_step, double_q=double_q,
            huber_delta=delta)
        n_agents = len(self.policy_tag_to_agent_id_map[policy])
        rows = self._init_replay(policy)
        if self.prioritized is not None:
            store = self.priority_stores[policy] = PrioritizedReplay(
                self.ring_capacity, self.num_envs * n_agents, self.n_step, rows,
                self.prioritized["alpha"], self.prioritized["epsilon"],
                next(q_net.parameters()).device)
            if self.verbose:
                print(f"[Device {self.device_id}]: priority store of policy '{policy}': "
                      f"{store.leaves.numel()} windows, a sum tree of {store.levels} levels, "
                      f"{store.nbytes()} bytes on the device")
        if implicit:
            dev = next(q_net.parameters()).device
            self.iqn_taus[policy] = torch.zeros(
                rows, q_net.num_tau_samples + q_net.num_tau_prime_samples, device=dev)
            if self._tau_generator is None:
                self._tau_generator = torch.Generator(device=dev)
                self._tau_generator.manual_seed(self.seed)
        masked = q_net.masked                  # masked QR-DQN / IQN: the torch losses
        fused = (FusedNoisyUpdate if q_net.noisy else FusedDuelingUpdate if q_net.dueling
                 else (FusedMaskedC51Update if masked else FusedC51Update) if categorical
                 else FusedIQNUpdate if implicit else FusedQRDQNUpdate if quantile
                 else FusedBranchingDQNUpdate if branching
                 else FusedMaskedDQNUpdate if masked else FusedDQNUpdate)
        if fused.supported(algo, q_net, self.num_envs, n_agents, self.ring_capacity, rows):
            extra = (self.seed,) if q_net.noisy else ()
            self.fused_updates[policy] = fused(
                algo, q_net, self.target_q_models[policy], self.num_envs, n_agents,
                self.ring_capacity, rows, *extra)

    def _make_engine(self, use_cuda_graph):
        engine = RingRolloutEngine(
            self.cuda_envs, self.q_models, self.policy_tag_to_agent_id_map,
            self.cuda_sample_controller, self.training_batch_size_per_env,
            ring_capacity=self.ring_capacity)
        engine.noise_seed = self.seed          # acting noise: this rank's seed
        return engine

    # ------------------------------------------------------------------ update
    def _ring_state(self):
        return self.engine.ring_cursor, self.engine.ring_filled

    def _generate_rollout_batch(self):
        before = self._ring_state()
        params = super()._generate_rollout_batch()
        self.last_epsilon = params["epsilon"]
        for store in self.priority_stores.values():     # warm-up rollouts included
            store.admit(before, self._ring_state())
        return params

    def _update_model_params(self, iteration):
        metrics_dict = super()._update_model_params(iteration)
        if self.last_epsilon is not None:      # the rollout's exploration rate
            for metrics in metrics_dict.values():
                metrics["Epsilon"] = float(self.last_epsilon)
        for policy, metrics in metrics_dict.items():
            noisy = self.q_models[policy].noisy_layers()
            if noisy:                          # how far the head has annealed its noise
                with torch.no_grad():
                    total = sum(L.weight_sigma.abs().double().sum() for L in noisy)
                    count = sum(L.weight_sigma.numel() for L in noisy)
                metrics["Noisy sigma"] = float(total / count)
            store = self.priority_stores.get(policy)
            if store is not None and "Q loss" in metrics:   # the last update's sample
                metrics["Priority beta"] = float(store.beta)
                metrics["Mean IS weight"] = float(store.weights.double().mean())
                metrics["Max priority"] = float(store.p_max)
        return metrics_dict

    def _sample_replay_windows(self, policy):
        """Uniform windows (TrainerDDPG), or with prioritized replay stratified proportional
        ones and their importance-sampling weights (two launches, no host wait)."""
        store = self.priority_stores.get(policy)
        if store is None:
            return super()._sample_replay_windows(policy)
        self.replay_draws += 1
        store.set_beta(self.prioritized["beta"].get_param_value(self.current_timestep[policy]))
        store.sample(self.replay_windows[policy], self.seed, self.replay_draws)

    def _one_update(self, logging_flag, step_info):
        """The Q gradient of every trained policy, one optimizer step, and the targets' tracking
        on every target_update_period-th update; returns the loss metrics (filled when
        logging_flag)."""
        loss_metrics = {}
        for policy in self.policies_to_train:
            self.update_count[policy] += 1
            self._sample_replay_windows(policy)
            if policy in self.iqn_taus:
                self.iqn_taus[policy].uniform_(generator=self._tau_generator)
            fused = self.fused_updates.get(policy)
            if fused is not None and self.trainers[policy].use_fused_update:
                loss_metrics[policy] = self._fused_q_gradients(policy, fused, logging_flag)
            else:
                loss_metrics[policy] = self._torch_q_gradients(policy, logging_flag)
            store = self.priority_stores.get(policy)
            if store is not None:
                eng = self.engine
                oldest = eng.ring_cursor if eng.ring_filled == eng.ring_capacity else 0
                store.set_priorities(self.replay_windows[policy], store.q_values, store.returns,
                                     oldest, eng.ring_filled)
        step_info.update(self._optimizer_step(loss_metrics, logging_flag))
        for policy in loss_metrics:
            if self.update_count[policy] % self.target_update_period[policy] == 0:
                soft_update(self.target_q_models[policy], self.q_models[policy],
                            self.tau[policy])
        return loss_metrics

    def _torch_q_gradients(self, policy, logging_flag):
        """The Q gradient by torch autograd on the gathered windows (the loss of
        wdb_dqn_update_sampled, or of wdb_qr_dqn_update_sampled / wdb_iqn_update_sampled /
        wdb_c51_update_sampled for a distributional network), accumulated into the arena's .grad views."""
        algo = self.trainers[policy]
        store = self.priority_stores.get(policy)
        nets = (self.q_models[policy], self.target_q_models[policy])
        noisy = [L for net in nets for L in net.noisy_layers()]
        for row, net in enumerate(nets):       # FusedNoisyUpdate's sample of this update
            if net.noisy:
                draw_noise(net, self.seed, NOISY_UPDATE, self.update_count[policy], row0=row)
        for L in noisy:
            L.noise = (L.noise_in, L.noise_out)
        try:
            loss, q, returns = algo.loss(*nets, *self._gather_windows(policy),
                                         weights=None if store is None else store.weights,
                                         boot_mask=self._gather_boot_mask(policy),
                                         **self._levels(policy))
        finally:
            for L in noisy:
                L.noise = None
        if store is not None:                  # the inputs of the new priorities
            store.q_values.copy_(q.detach())
            store.returns.copy_(returns)
        self.optimizers[policy].zero_grad()
        loss.backward()
        if not logging_flag:
            return {}
        return algo.loss_metrics(loss.item(), q.detach().double().mean(), returns)

    def _fused_q_gradients(self, policy, fused, logging_flag):
        """The same gradient from the native pass (FusedDQNUpdate, FusedQRDQNUpdate,
        FusedIQNUpdate, FusedC51Update, FusedDuelingUpdate, FusedNoisyUpdate or
        FusedBranchingDQNUpdate), written straight
        into the arena's .grad views; the host waits only on logging iterations (metrics)."""
        eng = self.engine
        outputs, weights = None, None
        store = self.priority_stores.get(policy)
        if store is not None:                  # the weighted pass; Q and R feed the priorities
            outputs, weights = (store.q_values, store.returns), store.weights
        elif logging_flag:
            dev = fused.sums.device
            outputs = (torch.empty(fused.rows, device=dev), torch.empty(fused.rows, device=dev))
        sums = fused.launch(eng._tensor(f"{_PROCESSED_OBSERVATIONS}_batch_{policy}"),
                            eng._tensor(f"{_ACTIONS}_batch_{policy}"),
                            eng._tensor(f"{_REWARDS}_batch_{policy}"),
                            eng._tensor(f"{_DONE_FLAGS}_batch"), self.replay_windows[policy],
                            outputs, weights, **self._levels(policy),
                            **({"update": self.update_count[policy]}
                               if isinstance(fused, FusedNoisyUpdate) else {}),
                            **({"action_mask": eng._tensor(f"{_ACTION_MASK}_batch_{policy}")}
                               if self.q_models[policy].masked else {}))
        if not logging_flag:
            return {}
        s = sums.tolist()
        return self.trainers[policy].loss_metrics(s[0] / fused.rows, s[1] / fused.rows,
                                                  outputs[1])

    def _gather_boot_mask(self, policy):
        """For an action-masked policy, obs' own mask [B, A] of the sampled windows: the ring's
        action_mask_batch_{p} row at each window's slot(n_step), the row the masked native
        passes read; None otherwise."""
        if not self.q_models[policy].masked:
            return None
        C = self.ring_capacity
        windows = self.replay_windows[policy].long()
        slot = (windows[:, 0] + self.n_step) % C
        mask = self.engine._tensor(f"{_ACTION_MASK}_batch_{policy}")
        return mask.reshape(C, -1, mask.shape[-1])[slot, windows[:, 1]]

    def _levels(self, policy):
        """IQN's levels of this update, as the `taus` argument of its loss and its native pass
        (nothing for the other Q networks)."""
        taus = self.iqn_taus.get(policy)
        return {} if taus is None else {"taus": taus}

    # ------------------------------------------------------------------ checkpoints
    def _checkpointed_networks(self):
        return [(policy, f"{policy}_q", model) for policy, model in self.q_models.items()]

    def _load_policy_checkpoint(self, policy, path):
        if not path:
            return
        if not isinstance(path, str):
            raise ValueError(f"DQN's model_ckpt_filepath is one path, got {path!r}")
        assert os.path.isfile(path), "Invalid model checkpoint path!"
        self.q_models[policy].load_state_dict(torch.load(path, map_location="cpu"))
        hard_update(self.target_q_models[policy], self.q_models[policy])
        self.current_timestep[policy] = self._checkpoint_timestep(path)
