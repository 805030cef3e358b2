"""TrainerDiscreteSAC: discrete-action SAC (algorithms/sac_discrete.py) for envs with one Discrete
action -- a policy with `algorithm: "DiscreteSAC"` in its run config (CartPole, MountainCar,
Acrobot).  TrainerSAC's temperature (`alpha`, `autotune_alpha`, `target_entropy`, `lr.alpha`),
twin critics and their targets, joint critic FlatAdam, the split `lr` / `model` entries, `tau`,
`gamma`, `clip_grad_norm` and checkpoints; TrainerDDPG's replay buffer, which is required
(`replay_slots_per_env`: the passes read sampled windows only).  What differs:

  * the actor is a `fully_connected_actor` on one Discrete(A) head (a softmax policy with no
    value head), sampled categorically in the rollout -- the one-launch softmax kind of
    wdb_single_agent_rollout, or the per-step path's sampler -- and played as argmax pi by the
    evaluator; there is no target actor;
  * the critics are two `fully_connected_q` networks (plain: no dueling, noisy, masked,
    quantile, IQN or categorical head) with A outputs each;
  * the update draws no noise: the expectation over actions is exact.

Per policy and update: the windows (1 launch); the critic gradients
(wdb_sac_discrete_critic_update_sampled, 2 launches, or torch autograd for the shapes it does not
take) -> all-reduce -> clipping + Adam of the twin critic; the actor gradient through both
just-updated critics (wdb_sac_discrete_actor_update_sampled, 2 launches, or torch) and the
log_alpha gradient -> all-reduce -> clipping + Adam of the actor, Adam of log_alpha; the two
target critics track their critics with `tau`.  On one GPU the host waits only on logging
iterations.
"""
import torch

from warp_drive_b200.training.algorithms.fused_sac_discrete import FusedDiscreteSACUpdate
from warp_drive_b200.training.algorithms.sac_discrete import (DiscreteSAC, torch_actor_loss,
                                                              torch_sampled_critic_loss)
from warp_drive_b200.training.models.fully_connected_actor_critic import ActorAsPolicy
from warp_drive_b200.training.trainer_ddpg import RingRolloutEngine, hard_update, soft_update
from warp_drive_b200.training.trainer_sac import Temperature, TrainerSAC
from warp_drive_b200.training.utils.data_loader import dict_observation_keys
from warp_drive_b200.utils.constants import Constants

_ACTIONS = Constants.ACTIONS
_REWARDS = Constants.REWARDS
_DONE_FLAGS = Constants.DONE_FLAGS
_PROCESSED_OBSERVATIONS = Constants.PROCESSED_OBSERVATIONS


class TrainerDiscreteSAC(TrainerSAC):
    """TrainerSAC's setup and checkpoints with a categorical actor, plain Q critics and the
    discrete SAC update over sampled replay windows."""

    # ------------------------------------------------------------------ setup
    def _batch_slots_per_env(self, trainer_config):
        slots = super()._batch_slots_per_env(trainer_config)
        if self.replay is None:
            raise ValueError("discrete SAC trains from a replay buffer: set the trainer key "
                             "replay_slots_per_env")
        return slots

    def _initialize_policy_model(self, policy):
        from warp_drive_b200.training.models.fully_connected_actor_critic import (
            FullyConnectedActor)
        from warp_drive_b200.training.models.fully_connected_q import FullyConnectedQ

        c = self._get_config(["policy", policy])
        if c.get("algorithm") != "DiscreteSAC":
            raise ValueError(f"TrainerDiscreteSAC trains algorithm DiscreteSAC, policy "
                             f"'{policy}' has '{c.get('algorithm')}'")
        if self.sample_params_schedules:
            raise ValueError("discrete SAC samples its own softmax policy: sampler params "
                             f"{sorted(self.sample_params_schedules)} are not taken")
        actor_cfg, critic_cfg = self._split(policy, "model")
        actor = self.actor_models[policy] = self._build_model(policy, actor_cfg)
        if type(actor) is not FullyConnectedActor:
            raise ValueError("discrete SAC's model.actor is a `fully_connected_actor`, got "
                             f"'{actor_cfg.get('type')}'")
        if actor.is_deterministic or len(actor.output_dims) != 1:
            raise ValueError("discrete SAC takes an action space of one Discrete head, got "
                             f"head sizes {list(actor.output_dims)}"
                             + (" of a Box space" if actor.is_deterministic else ""))
        if dict_observation_keys(actor.observation_space)[1]:
            raise ValueError("discrete SAC does not take an action_mask in the observation space")
        for online, target in ((self.critic_models, self.target_critic_models),
                               (self.critic2_models, self.target_critic2_models)):
            critic = online[policy] = self._build_model(policy, critic_cfg)
            if type(critic) is not FullyConnectedQ:
                raise ValueError("discrete SAC's model.critic is a plain `fully_connected_q`, got "
                                 f"'{critic_cfg.get('type')}'")
            for key in ("dueling", "noisy", "masked"):
                if getattr(critic, key):
                    raise ValueError(f"discrete SAC's critic takes no model.critic.{key}")
            if critic.output_dims[0] != actor.output_dims[0]:
                raise ValueError(f"the actor has {actor.output_dims[0]} actions and the critic "
                                 f"{critic.output_dims[0]}: they must agree")
            target[policy] = self._build_model(policy, critic_cfg)
            hard_update(target[policy], online[policy])
        self.temperatures[policy] = Temperature(c.get("alpha", 0.2))

    def _initialize_policy_algorithm(self, policy):
        c = self._get_config(["policy", policy])
        self.clip_grad_norm[policy] = c["clip_grad_norm"]
        if c["clip_grad_norm"]:
            self.max_grad_norm[policy] = c["max_grad_norm"]
        self.tau[policy] = c["tau"]
        actor = self.actor_models[policy]
        self.trainers[policy] = DiscreteSAC(
            discount_factor_gamma=c["gamma"], normalize_advantage=c["normalize_advantage"],
            normalize_return=c["normalize_return"], n_step=self.n_step,
            alpha=c.get("alpha", 0.2), autotune_alpha=c.get("autotune_alpha", True),
            target_entropy=c.get("target_entropy"), n_actions=int(actor.output_dims[0]))
        n_agents = len(self.policy_tag_to_agent_id_map[policy])
        rows = self._init_replay(policy)
        args = (self.num_envs, n_agents, self.ring_capacity, self.n_step)
        critic, critic2 = self.critic_models[policy], self.critic2_models[policy]
        if FusedDiscreteSACUpdate.supported(actor, critic, critic2, *args, rows):
            self.fused_updates[policy] = FusedDiscreteSACUpdate(
                actor, critic, critic2, self.target_critic_models[policy],
                self.target_critic2_models[policy], self.temperatures[policy].log_alpha, *args,
                gamma=c["gamma"], rows=rows)

    def _make_engine(self, use_cuda_graph):
        return RingRolloutEngine(
            self.cuda_envs, {p: ActorAsPolicy(self.actor_models[p]) for p in self.policies},
            self.policy_tag_to_agent_id_map, self.cuda_sample_controller,
            self.training_batch_size_per_env, ring_capacity=self.ring_capacity)

    # ------------------------------------------------------------------ update
    def _one_update(self, logging_flag, step_info):
        loss_metrics = {}
        for policy in self.policies_to_train:
            self._sample_replay_windows(policy)
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
        windows = self.replay_windows[policy]
        if fused is not None:
            outputs = None
            if logging_flag:
                outputs = tuple(torch.empty(fused.rows, device=windows.device) for _ in range(3))
            sums = fused.critic_launch(
                eng._tensor(f"{_PROCESSED_OBSERVATIONS}_batch_{policy}"),
                eng._tensor(f"{_ACTIONS}_batch_{policy}"),
                eng._tensor(f"{_REWARDS}_batch_{policy}"), eng._tensor(f"{_DONE_FLAGS}_batch"),
                windows, outputs)
            if not logging_flag:
                return {}
            s = sums.tolist()
            return algo.critic_metrics(s[0] / fused.rows, s[1] / fused.rows,
                                       outputs[0].double().mean(), outputs[2])
        l1, l2, q1, _, returns = torch_sampled_critic_loss(
            algo, self.actor_models[policy], self.target_critic_models[policy],
            self.target_critic2_models[policy], self.critic_models[policy],
            self.critic2_models[policy], self.temperatures[policy].log_alpha,
            *self._gather_windows(policy))
        self.critic_optimizers[policy].zero_grad()
        (l1 + l2).backward()
        if not logging_flag:
            return {}
        return algo.critic_metrics(l1.item(), l2.item(), q1.detach().double().mean(), returns)

    def _actor_gradients(self, policy, logging_flag):
        """The actor's gradient (through both critics as the critic step left them) into its
        .grad views, and log_alpha's; the actor and temperature metrics of a logging
        iteration."""
        eng, algo, fused = self.engine, self.trainers[policy], self._fused(policy)
        log_alpha = self.temperatures[policy].log_alpha
        windows = self.replay_windows[policy]
        if fused is not None:
            sums = fused.actor_launch(eng._tensor(f"{_PROCESSED_OBSERVATIONS}_batch_{policy}"),
                                      windows)
            rows, sum_m, sum_log_pi = fused.rows, sums[2], sums[3]
            actor_loss = None
        else:
            self.actor_optimizers[policy].zero_grad()
            actor_loss, pm, plp = torch_actor_loss(
                algo, self.actor_models[policy], self.critic_models[policy],
                self.critic2_models[policy], log_alpha, self._gather_windows(policy)[0])
            actor_loss.backward(inputs=list(self.actor_models[policy].parameters()))
            rows, sum_m, sum_log_pi = plp.numel(), pm.double().sum(), plp.double().sum()
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
            actor_loss_value = (alpha_value * float(sum_log_pi) - float(sum_m)) / rows
        else:
            actor_loss_value = actor_loss.item()
        alpha_loss = -float(log_alpha.detach()) * (mean_log_pi + algo.target_entropy)
        return algo.actor_metrics(actor_loss_value, mean_log_pi, alpha_value, alpha_loss)
