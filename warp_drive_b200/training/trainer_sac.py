"""TrainerSAC: SAC (algorithms/sac.py) for continuous (Box) action spaces -- a policy with
`algorithm: "SAC"` in its run config.  TrainerTD3's ring, twin critics and their targets, joint
critic FlatAdam, `n_step`, `tau`, `gamma`, the split `lr` / `model` entries and
`clip_grad_norm`; what differs:

  * the actor is a tanh-squashed Gaussian (`fully_connected_sac_actor`) sampled in the rollout
    by wdb_sample_squashed_gaussian on the per-step path (no OU noise: SAC takes no sampler
    params); the evaluator plays scale * tanh(mu) + bias;
  * there is no target actor: the critic's bootstrap samples the current actor;
  * log_alpha (alpha = exp(log_alpha)) is a parameter in the gradient arena, so the one
    all-reduce covers it on several GPUs, stepped by its own FlatAdam without clipping (config
    keys `alpha`, `autotune_alpha`, `target_entropy`, `lr.alpha`).

Per policy and update:
  1. critic gradients (wdb_sac_critic_update, or torch autograd for the shapes it does not
     take) -> all-reduce -> clipping + Adam of the twin critic;
  2. actor gradients through both just-updated critics (wdb_sac_actor_update, or torch) and
     the log_alpha gradient -> all-reduce -> clipping + Adam of the actor, Adam of log_alpha;
  3. the two target critics track their critics with `tau`.
The critic's eps' and the actor's eps are drawn per update from a CUDA generator seeded from
the trainer seed into two preallocated [valid, E, Np, A] buffers, indexed by logical window; the
fused and the torch update read the same buffers.  On one GPU the host waits only on logging
iterations.  With a replay buffer (trainer_ddpg.py) every iteration runs `updates_per_iteration`
such updates, each over its own sampled windows, and the noise buffers are [B, A].
"""
import math
import os

import torch
from torch import nn

from warp_drive_b200.training.algorithms.fused_sac import FusedSACUpdate, fused_sac_supported
from warp_drive_b200.training.algorithms.sac import (SAC, torch_actor_loss, torch_critic_loss,
                                                     torch_sampled_critic_loss)
from warp_drive_b200.training.trainer_ddpg import hard_update, soft_update
from warp_drive_b200.training.trainer_td3 import TrainerTD3
from warp_drive_b200.training.utils.param_scheduler import ParamScheduler
from warp_drive_b200.utils.constants import Constants

_ACTIONS = Constants.ACTIONS
_REWARDS = Constants.REWARDS
_DONE_FLAGS = Constants.DONE_FLAGS
_PROCESSED_OBSERVATIONS = Constants.PROCESSED_OBSERVATIONS


class Temperature(nn.Module):
    """SAC's entropy temperature: alpha = exp(log_alpha), log_alpha a parameter of shape [1]."""

    def __init__(self, alpha):
        super().__init__()
        if not alpha > 0:
            raise ValueError(f"alpha must be > 0, got {alpha}")
        self.log_alpha = nn.Parameter(torch.tensor([math.log(float(alpha))]))


class TrainerSAC(TrainerTD3):
    """TrainerTD3's setup without a target actor, with a temperature per policy, SAC's update
    and checkpoints `{policy}_actor_{t}`, `{policy}_critic_{t}`, `{policy}_critic2_{t}` and
    `{policy}_alpha_{t}`."""

    # the evaluator plays the squashed mean
    _test_sample_params = {"use_argmax": True}

    # ------------------------------------------------------------------ setup
    def _create_network_dicts(self):
        super()._create_network_dicts()
        self.temperatures, self.alpha_optimizers, self.alpha_lr_schedules = {}, {}, {}
        self.critic_noise, self.actor_noise = {}, {}

    def _initialize_policy_model(self, policy):
        c = self._get_config(["policy", policy])
        if c.get("algorithm") == "SAC" and self.sample_params_schedules:
            raise ValueError("SAC samples its own squashed Gaussian: sampler params "
                             f"{sorted(self.sample_params_schedules)} are not taken")
        actor_cfg, critic_cfg = self._split(policy, "model")
        self.actor_models[policy] = self._build_model(policy, actor_cfg)
        if not getattr(self.actor_models[policy], "is_squashed_gaussian", False):
            raise ValueError("SAC's actor is a `fully_connected_sac_actor`, got "
                             f"'{actor_cfg.get('type')}'")
        for online, target in ((self.critic_models, self.target_critic_models),
                               (self.critic2_models, self.target_critic2_models)):
            online[policy] = self._build_model(policy, critic_cfg)
            target[policy] = self._build_model(policy, critic_cfg)
            hard_update(target[policy], online[policy])
        self.temperatures[policy] = Temperature(c.get("alpha", 0.2))

    def _trained_networks(self, policy):
        return [self.actor_models[policy], self.critic_models[policy],
                self.critic2_models[policy], self.temperatures[policy]]

    def _all_networks(self, policy):
        return self._trained_networks(policy) + [
            self.target_critic_models[policy], self.target_critic2_models[policy]]

    def _initialize_optimizer(self, policy):
        super()._initialize_optimizer(policy)
        lr = self._get_config(["policy", policy, "lr"])
        alpha_lr = lr.get("alpha", lr["actor"]) if isinstance(lr, dict) and "actor" in lr else lr
        self.alpha_lr_schedules[policy] = ParamScheduler(alpha_lr)
        self.alpha_optimizers[policy] = self._flat_adam(
            self.temperatures[policy],
            self.alpha_lr_schedules[policy].get_param_value(self.current_timestep[policy]))

    def _optimizers_of(self, policy):
        return super()._optimizers_of(policy) + [
            (" (Alpha)", self.alpha_optimizers[policy], self.alpha_lr_schedules[policy])]

    def _initialize_policy_algorithm(self, policy):
        c = self._get_config(["policy", policy])
        assert c["algorithm"] == "SAC"
        self.clip_grad_norm[policy] = c["clip_grad_norm"]
        if c["clip_grad_norm"]:
            self.max_grad_norm[policy] = c["max_grad_norm"]
        self.tau[policy] = c["tau"]
        actor = self.actor_models[policy]
        A = int(actor.output_dims[0])
        algo = self.trainers[policy] = SAC(
            discount_factor_gamma=c["gamma"], normalize_advantage=c["normalize_advantage"],
            normalize_return=c["normalize_return"], n_step=self.n_step,
            alpha=c.get("alpha", 0.2), autotune_alpha=c.get("autotune_alpha", True),
            target_entropy=c.get("target_entropy"), action_dim=A)
        n_agents = len(self.policy_tag_to_agent_id_map[policy])
        dev = next(actor.parameters()).device
        valid = self.ring_capacity - self.n_step + 1
        rows = self._init_replay(policy)
        shape = self._noise_shape(rows, valid, n_agents, A)
        self.critic_noise[policy] = torch.zeros(shape, device=dev)
        self.actor_noise[policy] = torch.zeros(shape, device=dev)
        self.bootstrap_index[policy] = torch.tensor(algo.bootstrap_slots(self.ring_capacity),
                                                    device=dev)
        self.update_count[policy] = 0
        if self._noise_generator is None:
            self._noise_generator = torch.Generator(device=dev)
            self._noise_generator.manual_seed(self.seed)
        args = (self.num_envs, n_agents, self.ring_capacity, self.n_step)
        critic, critic2 = self.critic_models[policy], self.critic2_models[policy]
        if fused_sac_supported(algo, actor, critic, critic2, *args, replay_rows=rows):
            self.fused_updates[policy] = FusedSACUpdate(
                actor, critic, critic2, self.target_critic_models[policy],
                self.target_critic2_models[policy], self.temperatures[policy].log_alpha, *args,
                gamma=c["gamma"], replay_rows=rows)

    # ------------------------------------------------------------------ update
    def _one_update(self, logging_flag, step_info):
        loss_metrics = {}
        for policy in self.policies_to_train:
            self.update_count[policy] += 1
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
            for target, source in ((self.target_critic_models, self.critic_models),
                                   (self.target_critic2_models, self.critic2_models)):
                soft_update(target[policy], source[policy], self.tau[policy])
        return loss_metrics

    def _critic_gradients(self, policy, logging_flag):
        """Both critics' gradients into the arena's .grad views; the critic metrics of a
        logging iteration."""
        eng, algo, fused = self.engine, self.trainers[policy], self._fused(policy)
        log_alpha = self.temperatures[policy].log_alpha
        windows = self.replay_windows.get(policy)
        if fused is not None:
            rewards = eng._tensor(f"{_REWARDS}_batch_{policy}")
            actions = eng._tensor(f"{_ACTIONS}_batch_{policy}")
            outputs = None
            if logging_flag:
                shape = (fused.valid,) + tuple(rewards.shape[1:]) if windows is None else (
                    1, fused.rows, 1)
                outputs = tuple(torch.empty(shape, device=rewards.device) for _ in range(3))
            sums = fused.critic_launch(
                eng._tensor(f"{_PROCESSED_OBSERVATIONS}_batch_{policy}"), actions, rewards,
                eng._tensor(f"{_DONE_FLAGS}_batch"), eng.ring_cursor, self.critic_noise[policy],
                outputs, windows=windows)
            if not logging_flag:
                return {}
            s = sums.tolist()
            q1, _, returns = outputs
            if windows is not None:
                return self._replay_critic_metrics(policy, s[0] / fused.rows, s[1] / fused.rows,
                                                   q1, returns)
            return algo.loss_metrics(s[0] / fused.rows, s[1] / fused.rows, rewards, actions, q1,
                                     returns)
        if windows is not None:
            l1, l2, q1, _, returns = torch_sampled_critic_loss(
                algo, self.actor_models[policy], self.target_critic_models[policy],
                self.target_critic2_models[policy], self.critic_models[policy],
                self.critic2_models[policy], log_alpha, *self._gather_windows(policy),
                self.critic_noise[policy])
            self.critic_optimizers[policy].zero_grad()
            (l1 + l2).backward()
            if not logging_flag:
                return {}
            return self._replay_critic_metrics(policy, l1.item(), l2.item(),
                                               q1.detach()[None, :, None],
                                               returns[None, :, None])
        rewards = eng.unroll(f"{_REWARDS}_batch_{policy}")
        actions = eng.unroll(f"{_ACTIONS}_batch_{policy}")
        l1, l2, q1, _, returns = torch_critic_loss(
            algo, self.actor_models[policy], self.target_critic_models[policy],
            self.target_critic2_models[policy], self.critic_models[policy],
            self.critic2_models[policy], log_alpha,
            eng.unroll(f"{_PROCESSED_OBSERVATIONS}_batch_{policy}"), actions, rewards,
            eng.unroll(f"{_DONE_FLAGS}_batch"), self.critic_noise[policy],
            self.bootstrap_index[policy])
        self.critic_optimizers[policy].zero_grad()
        (l1 + l2).backward()
        if not logging_flag:
            return {}
        return algo.loss_metrics(l1.item(), l2.item(), rewards, actions, q1.detach(), returns)

    def _actor_gradients(self, policy, logging_flag):
        """The actor's gradient (through both critics as the critic step left them) into its
        .grad views, and log_alpha's; the actor and temperature metrics of a logging
        iteration."""
        eng, algo, fused = self.engine, self.trainers[policy], self._fused(policy)
        obs_name = f"{_PROCESSED_OBSERVATIONS}_batch_{policy}"
        log_alpha = self.temperatures[policy].log_alpha
        windows = self.replay_windows.get(policy)
        if fused is not None:
            sums = fused.actor_launch(eng._tensor(obs_name), eng.ring_cursor,
                                      self.actor_noise[policy], windows=windows)
            rows = fused.rows
            sum_q, sum_log_pi = sums[2], sums[3]
            alpha = log_alpha.detach().exp()
            actor_loss = None
        else:
            actor = self.actor_models[policy]
            if windows is not None:
                obs_rows = self._gather_windows(policy)[0]
            else:
                obs_rows = eng.unroll(obs_name)[:self.actor_noise[policy].shape[0]]
            self.actor_optimizers[policy].zero_grad()
            loss, q, log_pi = torch_actor_loss(
                algo, actor, self.critic_models[policy], self.critic2_models[policy], log_alpha,
                obs_rows, self.actor_noise[policy])
            loss.backward(inputs=list(actor.parameters()))
            rows = log_pi.numel()
            sum_log_pi = log_pi.detach().double().sum()
            actor_loss = loss
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
    def _checkpointed_networks(self):
        return super()._checkpointed_networks() + [
            (policy, f"{policy}_alpha", model) for policy, model in self.temperatures.items()]

    def _load_policy_checkpoint(self, policy, paths):
        if not (isinstance(paths, dict) and paths.get("actor") and paths.get("critic")
                and paths.get("critic2")):
            return
        names = ["actor", "critic", "critic2"] + (["alpha"] if paths.get("alpha") else [])
        steps = set()
        for k in names:
            assert os.path.isfile(paths[k]), f"Invalid {k} model checkpoint path!"
            steps.add(self._checkpoint_timestep(paths[k]))
        assert len(steps) == 1, f"The timesteps of the {names} checkpoints differ: {steps}"
        nets = {"actor": self.actor_models, "critic": self.critic_models,
                "critic2": self.critic2_models, "alpha": self.temperatures}
        for k in names:
            nets[k][policy].load_state_dict(torch.load(paths[k], map_location="cpu"))
        hard_update(self.target_critic_models[policy], self.critic_models[policy])
        hard_update(self.target_critic2_models[policy], self.critic2_models[policy])
        self.current_timestep[policy] = steps.pop()
