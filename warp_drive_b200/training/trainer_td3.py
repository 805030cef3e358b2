"""TrainerTD3: TD3 (algorithms/td3.py) for continuous (Box) action spaces -- a policy with
`algorithm: "TD3"` in its run config.  Everything but the update is TrainerDDPG's: the
constructor, the one-launch rollout with OU exploration noise, the replay ring, `n_step`, `tau`,
`gamma`, the split `lr` / `model` entries, `clip_grad_norm` and the evaluator.

Per policy: an actor, two critics and the three target networks; one FlatAdam for the actor and
one for the twin critic (both critics' parameters, clipped by their joint norm).  Update k of a
policy (k = 1, 2, ...):
  1. critic gradients (wdb_td3_critic_update, or torch autograd for the shapes it does not
     take) -> all-reduce -> clipping + Adam of the twin critic;
  2. if k % policy_delay == 0: actor gradients through the just-updated Q1
     (wdb_td3_actor_update, or torch) -> all-reduce -> clipping + Adam of the actor;
  3. on those updates only, the three targets track their networks with `tau`.
The target-policy noise is one draw of a CUDA generator seeded from the trainer seed per update
into a preallocated [valid, E, Np, A] buffer, indexed by logical window; the fused and the
torch update read the same buffer.  On one GPU the host waits only on logging iterations.
With a replay buffer (trainer_ddpg.py) k counts the `updates_per_iteration` updates of every
iteration, each over its own sampled windows, and the noise buffer is [B, A], one row per
sampled window.
"""
import os

import torch
from torch import nn

from warp_drive_b200.training.algorithms.fused_td3 import FusedTD3Update, fused_td3_supported
from warp_drive_b200.training.algorithms.td3 import (TD3, torch_actor_loss, torch_critic_loss,
                                                     torch_sampled_critic_loss)
from warp_drive_b200.training.trainer_ddpg import TrainerDDPG, hard_update, soft_update
from warp_drive_b200.utils.constants import Constants

_ACTIONS = Constants.ACTIONS
_REWARDS = Constants.REWARDS
_DONE_FLAGS = Constants.DONE_FLAGS
_PROCESSED_OBSERVATIONS = Constants.PROCESSED_OBSERVATIONS


class TrainerTD3(TrainerDDPG):
    """TrainerDDPG with a second critic (and its target), TD3's update and checkpoints
    `{policy}_actor_{t}`, `{policy}_critic_{t}` (Q1, loadable as a DDPG critic) and
    `{policy}_critic2_{t}`."""

    # ------------------------------------------------------------------ setup
    def _create_network_dicts(self):
        super()._create_network_dicts()
        self.critic2_models, self.target_critic2_models = {}, {}
        self.target_noise, self.bootstrap_index, self.update_count = {}, {}, {}
        self._noise_generator = None

    def _initialize_policy_model(self, policy):
        super()._initialize_policy_model(policy)
        _, critic_cfg = self._split(policy, "model")
        self.critic2_models[policy] = self._build_model(policy, critic_cfg)
        self.target_critic2_models[policy] = self._build_model(policy, critic_cfg)
        hard_update(self.target_critic2_models[policy], self.critic2_models[policy])

    def _trained_networks(self, policy):
        return [self.actor_models[policy], self.critic_models[policy],
                self.critic2_models[policy]]

    def _all_networks(self, policy):
        return self._trained_networks(policy) + [
            self.target_actor_models[policy], self.target_critic_models[policy],
            self.target_critic2_models[policy]]

    def _critic_optimized(self, policy):
        # the twin critic: one FlatAdam over both critics, clipped by their joint norm
        return nn.ModuleList([self.critic_models[policy], self.critic2_models[policy]])

    def _initialize_policy_algorithm(self, policy):
        c = self._get_config(["policy", policy])
        assert c["algorithm"] == "TD3"
        self.clip_grad_norm[policy] = c["clip_grad_norm"]
        if c["clip_grad_norm"]:
            self.max_grad_norm[policy] = c["max_grad_norm"]
        self.tau[policy] = c["tau"]
        algo = self.trainers[policy] = TD3(
            discount_factor_gamma=c["gamma"], normalize_advantage=c["normalize_advantage"],
            normalize_return=c["normalize_return"], n_step=self.n_step,
            target_noise=c.get("target_noise", 0.2),
            target_noise_clip=c.get("target_noise_clip", 0.5),
            policy_delay=c.get("policy_delay", 2))
        n_agents = len(self.policy_tag_to_agent_id_map[policy])
        actor = self.actor_models[policy]
        dev = next(actor.parameters()).device
        valid = self.ring_capacity - self.n_step + 1
        rows = self._init_replay(policy)
        self.target_noise[policy] = torch.zeros(
            self._noise_shape(rows, valid, n_agents, int(actor.output_dims[0])), device=dev)
        self.bootstrap_index[policy] = torch.tensor(algo.bootstrap_slots(self.ring_capacity),
                                                    device=dev)
        self.update_count[policy] = 0
        if self._noise_generator is None:
            self._noise_generator = torch.Generator(device=dev)
            self._noise_generator.manual_seed(self.seed)
        args = (self.num_envs, n_agents, self.ring_capacity, self.n_step)
        critic, critic2 = self.critic_models[policy], self.critic2_models[policy]
        if fused_td3_supported(algo, actor, critic, critic2, *args, replay_rows=rows):
            self.fused_updates[policy] = FusedTD3Update(
                algo, actor, critic, critic2, self.target_actor_models[policy],
                self.target_critic_models[policy], self.target_critic2_models[policy], *args,
                gamma=c["gamma"], replay_rows=rows)

    def _noise_shape(self, replay_rows, valid, n_agents, action_dim):
        """One row of noise per loss row: per window of the ring, or per sampled window."""
        if replay_rows is None:
            return (valid, self.num_envs, n_agents, action_dim)
        return (replay_rows, action_dim)

    # ------------------------------------------------------------------ update
    def _one_update(self, logging_flag, step_info):
        loss_metrics = {}
        for policy in self.policies_to_train:
            self.update_count[policy] += 1
            self._sample_replay_windows(policy)
            self.target_noise[policy].normal_(generator=self._noise_generator)
            loss_metrics[policy] = self._critic_gradients(policy, logging_flag)
        self._step(loss_metrics, 1, logging_flag, step_info)
        actors = [p for p in loss_metrics
                  if self.update_count[p] % self.trainers[p].policy_delay == 0]
        for policy in actors:
            loss_metrics[policy].update(self._actor_gradients(policy, logging_flag))
        if actors:
            self._step(actors, 0, logging_flag, step_info)
        for policy in actors:
            for target, source in (
                    (self.target_actor_models, self.actor_models),
                    (self.target_critic_models, self.critic_models),
                    (self.target_critic2_models, self.critic2_models)):
                soft_update(target[policy], source[policy], self.tau[policy])
        return loss_metrics

    def _step(self, stepped, which, logging_flag, step_info):
        """One all-reduce of the gradient arena, then clipping + Adam of network `which` (0:
        the actor, 1: the twin critic) of every policy in `stepped`; its gradient norm and
        learning rate go to step_info on a logging iteration."""
        if self.num_devices > 1 and stepped:
            self._allreduce_gradients()
        for policy in self.policies_to_train:
            norms, lrs = step_info.setdefault(policy, ({}, {}))
            if policy not in stepped:
                continue
            suffix, opt, _ = self._optimizers_of(policy)[which]
            if logging_flag:
                norms[f"Gradient norm{suffix}"] = sum(
                    p.grad.norm(2) for p in opt.param_list if p.grad is not None)
                lrs[f"Learning rate{suffix}"] = opt.param_groups[0]["lr"]
            opt.step(max_grad_norm=self.max_grad_norm[policy]
                     if self.clip_grad_norm[policy] else None)

    def _fused(self, policy):
        fused = self.fused_updates.get(policy)
        return fused if fused is not None and self.trainers[policy].use_fused_update else None

    def _critic_gradients(self, policy, logging_flag):
        """Both critics' gradients into the arena's .grad views; the critic metrics of a
        logging iteration."""
        eng, algo, fused = self.engine, self.trainers[policy], self._fused(policy)
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
                eng._tensor(f"{_DONE_FLAGS}_batch"), eng.ring_cursor, self.target_noise[policy],
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
                algo, self.target_actor_models[policy], self.target_critic_models[policy],
                self.target_critic2_models[policy], self.critic_models[policy],
                self.critic2_models[policy], *self._gather_windows(policy),
                self.target_noise[policy])
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
            algo, self.target_actor_models[policy], self.target_critic_models[policy],
            self.target_critic2_models[policy], self.critic_models[policy],
            self.critic2_models[policy], eng.unroll(f"{_PROCESSED_OBSERVATIONS}_batch_{policy}"),
            actions, rewards, eng.unroll(f"{_DONE_FLAGS}_batch"), self.target_noise[policy],
            self.bootstrap_index[policy])
        self.critic_optimizers[policy].zero_grad()
        (l1 + l2).backward()
        if not logging_flag:
            return {}
        return algo.loss_metrics(l1.item(), l2.item(), rewards, actions, q1.detach(), returns)

    def _replay_critic_metrics(self, policy, loss1, loss2, q1, returns):
        """The critic metrics of an update over sampled windows: q1 and returns [1, B, 1], the
        rewards and actions of the windows' first step."""
        _, actions, rewards, _, _ = self._gather_windows(policy)
        return self._batch_metrics(self.trainers[policy].loss_metrics(
            loss1, loss2, rewards[0][None, :, None], actions[None, :, None], q1, returns))

    def _actor_gradients(self, policy, logging_flag):
        """The actor's gradient (through Q1 as the critic step left it) into its .grad views
        only; the actor metrics of a logging iteration."""
        eng, algo, fused = self.engine, self.trainers[policy], self._fused(policy)
        obs_name = f"{_PROCESSED_OBSERVATIONS}_batch_{policy}"
        windows = self.replay_windows.get(policy)
        if fused is not None:
            sums = fused.actor_launch(eng._tensor(obs_name), eng.ring_cursor, windows=windows)
            return algo.actor_metrics(-float(sums[2]) / fused.rows) if logging_flag else {}
        actor = self.actor_models[policy]
        if windows is not None:
            obs_rows = self._gather_windows(policy)[0]
        else:
            obs_rows = eng.unroll(obs_name)[:self.target_noise[policy].shape[0]]
        loss, _ = torch_actor_loss(algo, actor, self.critic_models[policy], obs_rows)
        self.actor_optimizers[policy].zero_grad()
        loss.backward(inputs=list(actor.parameters()))
        return algo.actor_metrics(loss.item()) if logging_flag else {}

    # ------------------------------------------------------------------ checkpoints
    def _checkpointed_networks(self):
        return super()._checkpointed_networks() + [
            (policy, f"{policy}_critic2", model) for policy, model in self.critic2_models.items()]

    def _load_policy_checkpoint(self, policy, paths):
        super()._load_policy_checkpoint(policy, paths)
        if not (isinstance(paths, dict) and paths.get("actor") and paths.get("critic")
                and paths.get("critic2")):
            return
        assert os.path.isfile(paths["critic2"]), "Invalid critic2 model checkpoint path!"
        assert self._checkpoint_timestep(paths["critic2"]) == self.current_timestep[policy], (
            "The timestep is different between the actor model and the critic2 model ")
        self.critic2_models[policy].load_state_dict(
            torch.load(paths["critic2"], map_location="cpu"))
        hard_update(self.target_critic2_models[policy], self.critic2_models[policy])
