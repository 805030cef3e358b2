"""TrainerTQC: TQC (algorithms/tqc.py) for continuous (Box) action spaces -- a policy with
`algorithm: "TQC"` in its run config (Pendulum, ContinuousMountainCar).  TrainerSAC's actor
(`fully_connected_sac_actor`), rollout, temperature (`alpha`, `autotune_alpha`,
`target_entropy`, `lr.alpha`), noise buffers, the split `lr` / `model` entries, `tau`, `gamma`
and `clip_grad_norm`; TrainerDDPG's replay buffer, which is required (`replay_slots_per_env`:
the passes read sampled windows only).  What differs:

  * the critics are `n_critics` (policy key, default 2) `fully_connected_quantile_critic`
    networks of `num_quantiles` quantiles each (model key, default 25), held by one
    QuantileCritics module with its target copy: one FlatAdam steps them and clips them by their
    joint norm, and the `{policy}_critic_{t}` checkpoint holds all of them;
  * the bootstrap drops the `top_quantiles_to_drop_per_net` (policy key, default 2) largest
    atoms per critic from the pooled target atoms;
  * the actor follows the mean over all quantiles of all critics.

Per policy and update: the windows (1 launch); the critic gradients
(wdb_tqc_critic_update_sampled, 2 launches, or torch autograd for the shapes it does not take)
-> all-reduce -> clipping + Adam of the critics; the actor gradient through the just-updated
critics (wdb_tqc_actor_update_sampled, 2 launches, or torch) and the log_alpha gradient ->
all-reduce -> clipping + Adam of the actor, Adam of log_alpha; the target critics track their
critics with `tau`.  On one GPU the host waits only on logging iterations.
"""
import os

import torch

from warp_drive_b200.training.algorithms.fused_tqc import FusedTQCUpdate
from warp_drive_b200.training.algorithms.tqc import (TQC, torch_actor_loss,
                                                     torch_sampled_critic_loss)
from warp_drive_b200.training.models.fully_connected_actor_critic import QuantileCritics
from warp_drive_b200.training.trainer_ddpg import hard_update, soft_update
from warp_drive_b200.training.trainer_sac import Temperature, TrainerSAC
from warp_drive_b200.utils.constants import Constants

_ACTIONS = Constants.ACTIONS
_REWARDS = Constants.REWARDS
_DONE_FLAGS = Constants.DONE_FLAGS
_PROCESSED_OBSERVATIONS = Constants.PROCESSED_OBSERVATIONS


def _integer(v):
    return isinstance(v, int) and not isinstance(v, bool)


class TrainerTQC(TrainerSAC):
    """TrainerSAC's setup with M quantile critics, TQC's update over sampled replay windows and
    checkpoints `{policy}_actor_{t}`, `{policy}_critic_{t}` (all M critics) and
    `{policy}_alpha_{t}`."""

    # ------------------------------------------------------------------ setup
    def _batch_slots_per_env(self, trainer_config):
        slots = super()._batch_slots_per_env(trainer_config)
        if self.replay is None:
            raise ValueError("TQC trains from a replay buffer: set the trainer key "
                             "replay_slots_per_env")
        return slots

    def _initialize_policy_model(self, policy):
        c = self._get_config(["policy", policy])
        if c.get("algorithm") != "TQC":
            raise ValueError(f"TrainerTQC trains algorithm TQC, policy '{policy}' has "
                             f"'{c.get('algorithm')}'")
        if self.sample_params_schedules:
            raise ValueError("TQC samples its own squashed Gaussian: sampler params "
                             f"{sorted(self.sample_params_schedules)} are not taken")
        M = c.get("n_critics", 2)
        if not _integer(M) or M < 1:
            raise ValueError(f"n_critics must be an integer >= 1, got {M!r}")
        actor_cfg, critic_cfg = self._split(policy, "model")
        if actor_cfg.get("type") != "fully_connected_sac_actor":
            raise ValueError("TQC's model.actor is a `fully_connected_sac_actor`, got "
                             f"'{actor_cfg.get('type')}'")
        if critic_cfg.get("type") != "fully_connected_quantile_critic":
            raise ValueError("TQC's model.critic is a `fully_connected_quantile_critic`, got "
                             f"'{critic_cfg.get('type')}'")
        online = [self._build_model(policy, critic_cfg) for _ in range(M)]
        if not online[0].is_deterministic:
            raise ValueError("TQC takes a Box action space, got head sizes "
                             f"{list(online[0].output_dims)} of a discrete one")
        N = online[0].num_quantiles
        d = c.get("top_quantiles_to_drop_per_net", 2)
        if not _integer(d) or not 0 <= d <= N - 1:
            raise ValueError(f"top_quantiles_to_drop_per_net must be an integer in [0, "
                             f"num_quantiles - 1] = [0, {N - 1}], got {d!r}")
        self.actor_models[policy] = self._build_model(policy, actor_cfg)
        self.critic_models[policy] = QuantileCritics(online)
        self.target_critic_models[policy] = QuantileCritics(
            [self._build_model(policy, critic_cfg) for _ in range(M)])
        hard_update(self.target_critic_models[policy], self.critic_models[policy])
        self.temperatures[policy] = Temperature(c.get("alpha", 0.2))

    def _trained_networks(self, policy):
        return [self.actor_models[policy], self.critic_models[policy],
                self.temperatures[policy]]

    def _all_networks(self, policy):
        return self._trained_networks(policy) + [self.target_critic_models[policy]]

    def _critic_optimized(self, policy):
        # the M critics: one FlatAdam, clipped by their joint norm
        return self.critic_models[policy]

    def _initialize_policy_algorithm(self, policy):
        c = self._get_config(["policy", policy])
        self.clip_grad_norm[policy] = c["clip_grad_norm"]
        if c["clip_grad_norm"]:
            self.max_grad_norm[policy] = c["max_grad_norm"]
        self.tau[policy] = c["tau"]
        actor, critics = self.actor_models[policy], self.critic_models[policy]
        A = int(actor.output_dims[0])
        algo = self.trainers[policy] = TQC(
            discount_factor_gamma=c["gamma"], normalize_advantage=c["normalize_advantage"],
            normalize_return=c["normalize_return"], n_step=self.n_step,
            alpha=c.get("alpha", 0.2), autotune_alpha=c.get("autotune_alpha", True),
            target_entropy=c.get("target_entropy"), action_dim=A, n_critics=len(critics),
            n_quantiles=critics[0].num_quantiles,
            drop_per_net=c.get("top_quantiles_to_drop_per_net", 2))
        n_agents = len(self.policy_tag_to_agent_id_map[policy])
        rows = self._init_replay(policy)
        dev = next(actor.parameters()).device
        self.critic_noise[policy] = torch.zeros((rows, A), device=dev)
        self.actor_noise[policy] = torch.zeros((rows, A), device=dev)
        if self._noise_generator is None:
            self._noise_generator = torch.Generator(device=dev)
            self._noise_generator.manual_seed(self.seed)
        args = (self.num_envs, n_agents, self.ring_capacity, self.n_step)
        if FusedTQCUpdate.supported(algo, actor, critics, *args, rows):
            self.fused_updates[policy] = FusedTQCUpdate(
                algo, actor, critics, self.target_critic_models[policy],
                self.temperatures[policy].log_alpha, *args, rows)

    # ------------------------------------------------------------------ update
    def _one_update(self, logging_flag, step_info):
        loss_metrics = {}
        for policy in self.policies_to_train:
            self._sample_replay_windows(policy)
            self.critic_noise[policy].normal_(generator=self._noise_generator)
            self.actor_noise[policy].normal_(generator=self._noise_generator)
            loss_metrics[policy] = self._critic_gradients(policy, logging_flag)
        self._step(loss_metrics, 1, logging_flag, step_info)
        stepped = list(loss_metrics)
        for policy in stepped:
            loss_metrics[policy].update(self._actor_gradients(policy, logging_flag))
        if stepped:
            self._step(stepped, 0, logging_flag, step_info)
        for policy in stepped:
            if self.trainers[policy].autotune_alpha:
                self.alpha_optimizers[policy].step()
            soft_update(self.target_critic_models[policy], self.critic_models[policy],
                        self.tau[policy])
        return loss_metrics

    def _critic_gradients(self, policy, logging_flag):
        """The critics' gradients into the arena's .grad views; the critic metrics of a
        logging iteration."""
        eng, algo, fused = self.engine, self.trainers[policy], self._fused(policy)
        windows = self.replay_windows[policy]
        if fused is not None:
            outputs = None
            if logging_flag:
                outputs = tuple(torch.empty(fused.rows, device=windows.device) for _ in range(2))
            sums = fused.critic_launch(
                eng._tensor(f"{_PROCESSED_OBSERVATIONS}_batch_{policy}"),
                eng._tensor(f"{_ACTIONS}_batch_{policy}"),
                eng._tensor(f"{_REWARDS}_batch_{policy}"), eng._tensor(f"{_DONE_FLAGS}_batch"),
                self.critic_noise[policy], windows, outputs)
            if not logging_flag:
                return {}
            s = sums.tolist()
            pairs = fused.rows * 2 * algo.n_quantiles * algo.kept_atoms
            return algo.critic_metrics(s[0] / pairs, s[1] / fused.rows,
                                       outputs[1].double().mean())
        loss, theta, returns = torch_sampled_critic_loss(
            algo, self.actor_models[policy], self.target_critic_models[policy],
            self.critic_models[policy], self.temperatures[policy].log_alpha,
            *self._gather_windows(policy), self.critic_noise[policy])
        self.critic_optimizers[policy].zero_grad()
        loss.backward()
        if not logging_flag:
            return {}
        return algo.critic_metrics(loss.item(), theta.detach().double().mean(),
                                   returns.double().mean())

    def _actor_gradients(self, policy, logging_flag):
        """The actor's gradient (through the critics as the critic step left them) into its
        .grad views, and log_alpha's; the actor and temperature metrics of a logging
        iteration."""
        eng, algo, fused = self.engine, self.trainers[policy], self._fused(policy)
        log_alpha = self.temperatures[policy].log_alpha
        windows = self.replay_windows[policy]
        if fused is not None:
            sums = fused.actor_launch(eng._tensor(f"{_PROCESSED_OBSERVATIONS}_batch_{policy}"),
                                      self.actor_noise[policy], windows)
            rows, sum_q, sum_log_pi = fused.rows, sums[2], sums[3]
            actor_loss = None
        else:
            actor = self.actor_models[policy]
            self.actor_optimizers[policy].zero_grad()
            actor_loss, _, log_pi = torch_actor_loss(
                algo, actor, self.critic_models[policy], log_alpha,
                self._gather_windows(policy)[0], self.actor_noise[policy])
            actor_loss.backward(inputs=list(actor.parameters()))
            rows, sum_log_pi = log_pi.numel(), log_pi.detach().double().sum()
        grad = self.alpha_optimizers[policy].grads
        if algo.autotune_alpha:
            grad[:1].copy_(algo.alpha_grad(sum_log_pi, rows))
        else:
            grad.zero_()
        if not logging_flag:
            return {}
        mean_log_pi = float(sum_log_pi) / rows
        alpha_value = float(log_alpha.detach().exp())
        if actor_loss is None:
            actor_loss_value = (alpha_value * float(sum_log_pi) - float(sum_q)) / rows
        else:
            actor_loss_value = actor_loss.item()
        alpha_loss = -float(log_alpha.detach()) * (mean_log_pi + algo.target_entropy)
        return algo.actor_metrics(actor_loss_value, mean_log_pi, alpha_value, alpha_loss)

    # ------------------------------------------------------------------ checkpoints
    def _load_policy_checkpoint(self, policy, paths):
        if not (isinstance(paths, dict) and paths.get("actor") and paths.get("critic")):
            return
        names = ["actor", "critic"] + (["alpha"] if paths.get("alpha") else [])
        steps = set()
        for k in names:
            assert os.path.isfile(paths[k]), f"Invalid {k} model checkpoint path!"
            steps.add(self._checkpoint_timestep(paths[k]))
        assert len(steps) == 1, f"The timesteps of the {names} checkpoints differ: {steps}"
        nets = {"actor": self.actor_models, "critic": self.critic_models,
                "alpha": self.temperatures}
        for k in names:
            nets[k][policy].load_state_dict(torch.load(paths[k], map_location="cpu"))
        hard_update(self.target_critic_models[policy], self.critic_models[policy])
        self.current_timestep[policy] = steps.pop()
