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
"""
import json
import os
import random
import time

import numpy as np
import torch
import yaml
from torch import nn

from warp_drive_b200.managers.function_manager import CUDASampler
from warp_drive_b200.training.algorithms.ddpg import DDPG
from warp_drive_b200.training.algorithms.fused_ddpg import FusedDDPGUpdate, fused_ddpg_supported
from warp_drive_b200.training.models.fully_connected import ModelFactory
from warp_drive_b200.training.models.fully_connected_actor_critic import ActorAsPolicy
from warp_drive_b200.training.rollout import RolloutEngine
from warp_drive_b200.training.trainer import (
    _CONFIG_DIR, PerfStats, Trainer, recursive_merge_config_dicts, verbose_print)
from warp_drive_b200.training.utils.data_loader import (
    create_and_push_data_placeholders, validate_policy_map)
from warp_drive_b200.training.utils.flat_adam import FlatAdam
from warp_drive_b200.training.utils.param_scheduler import ParamScheduler
from warp_drive_b200.utils.constants import Constants

_ACTIONS = Constants.ACTIONS
_REWARDS = Constants.REWARDS
_DONE_FLAGS = Constants.DONE_FLAGS
_PROCESSED_OBSERVATIONS = Constants.PROCESSED_OBSERVATIONS
_EPSILON = 1e-10


def soft_update(target, source, tau):
    """target <- (1 - tau) * target + tau * source (trainer_ddpg.py:40-44), two fused launches."""
    tp, sp = list(target.parameters()), list(source.parameters())
    with torch.no_grad():
        torch._foreach_mul_(tp, 1.0 - tau)
        torch._foreach_add_(tp, sp, alpha=tau)


def hard_update(target, source):
    target.load_state_dict(source.state_dict())


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

    def step(self, t, **sample_params):
        if self.sa is not None and t >= 0 and self._sa_params_ok(sample_params):
            with torch.no_grad():
                self.sa.launch(1, t0=self._slot(t), **sample_params)
            return None
        return super().step(t, **sample_params)

    def evaluate_policies(self, t):
        return super().evaluate_policies(self._slot(t))

    def sample_actions(self, probs, t, **sample_params):
        return super().sample_actions(probs, self._slot(t), **sample_params)

    def bookkeep(self, t):
        return super().bookkeep(self._slot(t))

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
    def __init__(self, env_wrapper=None, config=None, policy_tag_to_agent_id_map=None,
                 create_separate_placeholders_for_each_policy=False,
                 obs_dim_corresponding_to_num_agents="first", num_devices=1, device_id=0,
                 results_dir=None, verbose=True):
        assert env_wrapper is not None and env_wrapper.env_backend != "cpu"
        assert config is not None
        assert not create_separate_placeholders_for_each_policy, (
            "separate per-policy step placeholders are not implemented in the native trainer")
        self.cuda_envs = env_wrapper
        self.verbose = verbose
        self.num_devices, self.device_id = num_devices, device_id

        with open(os.path.join(_CONFIG_DIR, "default_configs.yaml"), encoding="utf8") as fp:
            default = yaml.safe_load(fp)
        self.config = config
        config["trainer"] = recursive_merge_config_dicts(config["trainer"], default["trainer"])
        for key in config["policy"]:
            # actor / critic sub-dicts of `model` and `lr` are kept as given
            for k, v in default["policy"].items():
                config["policy"][key].setdefault(k, v)
        config["saving"] = recursive_merge_config_dicts(config["saving"], default["saving"])
        self.sample_params_schedules = {
            k: ParamScheduler(v) for k, v in config.get("sampler", {}).get("params", {}).items()}

        results_dir = results_dir or f"{time.time():10.0f}"
        s = config["saving"]
        self.save_dir = os.path.join(s["basedir"], s["name"], s["tag"], results_dir)
        os.makedirs(self.save_dir, exist_ok=True)
        with open(os.path.join(self.save_dir, "run_config.json"), "a+", encoding="utf8") as fp:
            json.dump(config, fp)
            fp.write("\n")

        self.policy_tag_to_agent_id_map = validate_policy_map(env_wrapper,
                                                              policy_tag_to_agent_id_map)
        self.policies = list(config["policy"].keys())
        assert set(self.policies) == set(self.policy_tag_to_agent_id_map.keys())
        self.policies_to_train = [p for p in self.policies if config["policy"][p]["to_train"]]

        t = config["trainer"]
        self.num_episodes = t["num_episodes"]
        self.training_batch_size = t["train_batch_size"]
        self.num_envs = t["num_envs"]
        assert self.num_envs == env_wrapper.n_envs
        self.training_batch_size_per_env = self.training_batch_size // self.num_envs
        assert self.training_batch_size_per_env > 0
        self.n_step = int(t.get("n_step", 1))
        assert self.n_step >= 1
        self.ring_capacity = self.training_batch_size_per_env + self.n_step - 1

        self.cuda_envs.reset_all_envs()
        self.cuda_sample_controller = CUDASampler(self.cuda_envs.cuda_function_manager)
        create_and_push_data_placeholders(
            env_wrapper=self.cuda_envs, action_sampler=self.cuda_sample_controller,
            policy_tag_to_agent_id_map=self.policy_tag_to_agent_id_map,
            obs_dim_corresponding_to_num_agents=obs_dim_corresponding_to_num_agents,
            training_batch_size_per_env=self.ring_capacity)
        seed = int(t.get("seed", np.int32(time.time()))) + self.device_id
        self.seed = seed
        self.cuda_sample_controller.init_random(seed)
        torch.manual_seed(seed)
        random.seed(seed)
        np.random.seed(seed)
        self.cuda_envs.init_reset_pool(seed + random.randint(1, 10000))

        self.total_steps = self.cuda_envs.episode_length * self.num_episodes
        self.num_iters = int(self.total_steps // self.training_batch_size)
        if self.num_iters == 0:
            raise ValueError("Not enough steps to even perform a single training iteration!. "
                             "Please increase the number of episodes or reduce the training "
                             "batch size.")

        self.actor_models, self.critic_models = {}, {}
        self.target_actor_models, self.target_critic_models = {}, {}
        self.actor_optimizers, self.critic_optimizers = {}, {}
        self.actor_lr_schedules, self.critic_lr_schedules = {}, {}
        self.tau, self.trainers = {}, {}
        self.clip_grad_norm, self.max_grad_norm, self.current_timestep = {}, {}, {}
        for policy in self.policies:
            self.current_timestep[policy] = 0
            self._initialize_policy_model(policy)
        self.load_model_checkpoint()
        for policy in self.policies:
            for group in (self.actor_models, self.critic_models, self.target_actor_models,
                          self.target_critic_models):
                group[policy].cuda()
        # ONE flat float32 arena for the parameters and one for the gradients of every actor
        # and critic (Trainer's layout): the multi-GPU all-reduce is one in-place NCCL call on
        # `_arena_grads`
        nets = [g[p] for p in self.policies for g in (self.actor_models, self.critic_models)]
        total = sum(FlatAdam.numel(m.parameters()) for m in nets)
        dev = next(nets[0].parameters()).device
        self._arena_params = torch.zeros(total, dtype=torch.float32, device=dev)
        self._arena_grads = torch.zeros(total, dtype=torch.float32, device=dev)
        self._arena_off = 0
        for policy in self.policies:
            self._initialize_optimizer(policy)
        self.fused_updates = {}
        for policy in self.policies_to_train:
            self._initialize_policy_algorithm(policy)
        if self.num_devices > 1:
            self._broadcast_parameters()

        # names the base class' helpers use (checkpointing is overridden below)
        self.models = self.actor_models
        self.engine = RingRolloutEngine(
            self.cuda_envs, {p: ActorAsPolicy(self.actor_models[p]) for p in self.policies},
            self.policy_tag_to_agent_id_map, self.cuda_sample_controller,
            self.training_batch_size_per_env, ring_capacity=self.ring_capacity)
        assert self.engine.continuous, "DDPG needs a continuous (Box) action space"
        self.perf_stats = PerfStats()
        self._flat_grad = None

    # ------------------------------------------------------------------ setup helpers
    def _split(self, policy, key):
        """(actor part, critic part) of a config entry that may or may not be split."""
        value = self._get_config(["policy", policy, key])
        if isinstance(value, dict) and "actor" in value and "critic" in value:
            return value["actor"], value["critic"]
        return value, value

    def _initialize_policy_model(self, policy):
        actor_cfg, critic_cfg = self._split(policy, "model")

        def build(cfg):
            model = ModelFactory.create(cfg["type"])(
                env=self.cuda_envs, model_config=cfg, policy=policy,
                policy_tag_to_agent_id_map=self.policy_tag_to_agent_id_map)
            if cfg.get("init_method") == "xavier":
                for m in model.modules():
                    if isinstance(m, nn.Linear):
                        nn.init.xavier_uniform_(m.weight)
            return model

        self.actor_models[policy] = build(actor_cfg)
        self.target_actor_models[policy] = build(actor_cfg)
        hard_update(self.target_actor_models[policy], self.actor_models[policy])
        self.critic_models[policy] = build(critic_cfg)
        self.target_critic_models[policy] = build(critic_cfg)
        hard_update(self.target_critic_models[policy], self.critic_models[policy])

    def _initialize_optimizer(self, policy):
        actor_lr, critic_lr = self._split(policy, "lr")
        self.actor_lr_schedules[policy] = ParamScheduler(actor_lr)
        self.critic_lr_schedules[policy] = ParamScheduler(critic_lr)
        ts = self.current_timestep[policy]

        def flat_adam(model, lr):
            n = FlatAdam.numel(model.parameters())
            lo = self._arena_off
            self._arena_off += n
            return FlatAdam(model.parameters(), lr=lr, arena=(
                self._arena_params[lo:lo + n], self._arena_grads[lo:lo + n]))

        self.actor_optimizers[policy] = flat_adam(
            self.actor_models[policy], self.actor_lr_schedules[policy].get_param_value(ts))
        self.critic_optimizers[policy] = flat_adam(
            self.critic_models[policy], self.critic_lr_schedules[policy].get_param_value(ts))

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
        if fused_ddpg_supported(self.trainers[policy], actor, critic, *args):
            self.fused_updates[policy] = FusedDDPGUpdate(
                actor, critic, self.target_actor_models[policy],
                self.target_critic_models[policy], *args, gamma=c["gamma"])

    # ------------------------------------------------------------------ multi-GPU
    def _trained_params(self):
        return [p for pol in self.policies_to_train
                for m in (self.actor_models[pol], self.critic_models[pol])
                for p in m.parameters()]

    def _broadcast_parameters(self):
        import torch.distributed as dist

        for pol in self.policies:
            for m in (self.actor_models[pol], self.critic_models[pol],
                      self.target_actor_models[pol], self.target_critic_models[pol]):
                for p in m.parameters():
                    dist.broadcast(p.data, src=0)

    # ------------------------------------------------------------------ update
    def _update_model_params(self, iteration):
        saving = self.config["saving"]
        logging_flag = (iteration % saving["metrics_log_freq"] == 0
                        or iteration == self.num_iters - 1)
        eng = self.engine
        metrics_dict = {}
        stepped = []
        if eng.isfull():
            for policy in self.policies_to_train:
                self.current_timestep[policy] += self.training_batch_size
                actor_lr = self.actor_lr_schedules[policy].get_param_value(
                    self.current_timestep[policy])
                critic_lr = self.critic_lr_schedules[policy].get_param_value(
                    self.current_timestep[policy])
                self.actor_optimizers[policy].param_groups[0]["lr"] = actor_lr
                self.critic_optimizers[policy].param_groups[0]["lr"] = critic_lr
                fused = self.fused_updates.get(policy)
                if fused is not None and self.trainers[policy].use_fused_update:
                    metrics = self._fused_gradients(policy, fused, logging_flag)
                else:
                    metrics = self._torch_gradients(policy, logging_flag)
                stepped.append((policy, metrics, actor_lr, critic_lr))
            if self.num_devices > 1 and stepped:
                self._allreduce_gradients()
        for policy, metrics, actor_lr, critic_lr in stepped:
            actor, critic = self.actor_models[policy], self.critic_models[policy]
            if logging_flag:
                metrics["Gradient norm (Actor)"] = float(sum(
                    p.grad.norm(2) for p in actor.parameters() if p.grad is not None))
                metrics["Gradient norm (Critic)"] = float(sum(
                    p.grad.norm(2) for p in critic.parameters() if p.grad is not None))
            # clip_grad_norm_ + Adam per network as two flat kernels each
            clip = self.max_grad_norm[policy] if self.clip_grad_norm[policy] else None
            self.actor_optimizers[policy].step(max_grad_norm=clip)
            self.critic_optimizers[policy].step(max_grad_norm=clip)
            soft_update(self.target_actor_models[policy], actor, self.tau[policy])
            soft_update(self.target_critic_models[policy], critic, self.tau[policy])
            if logging_flag:
                metrics.update({"Learning rate (Actor)": actor_lr,
                                "Learning rate (Critic)": critic_lr})
        if logging_flag:
            n_done = int(eng.num_completed_episodes)
            for policy in self.policies_to_train:
                m = next((x[1] for x in stepped if x[0] == policy), {})
                m.update({
                    "Current timestep": self.current_timestep[policy],
                    "Mean episodic reward":
                        float(eng.episodic_reward_sum[policy]) / (n_done + _EPSILON),
                    "Mean episodic steps": float(eng.episodic_step_sum) / (n_done + _EPSILON)})
                metrics_dict[policy] = m
            for policy in self.policies:
                eng.episodic_reward_sum[policy].zero_()
            eng.episodic_step_sum.zero_()
            eng.num_completed_episodes.zero_()
            if self.config["trainer"].get("evaluator"):
                reward_sum, step_sum = self.evaluate_episodes(scale=0)
                for policy in self.policies_to_train:
                    metrics_dict[policy].update({
                        "Mean episodic reward (test)": float(reward_sum[policy].mean()),
                        "Mean episodic steps (test)": float(step_sum[policy].float().mean())})
        return metrics_dict

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
        outputs = None
        if logging_flag:
            shape = (fused.valid,) + tuple(rewards.shape[1:])
            outputs = tuple(torch.empty(shape, device=rewards.device) for _ in range(3))
        sums = fused.launch(eng._tensor(f"{_PROCESSED_OBSERVATIONS}_batch_{policy}"), actions,
                            rewards, eng._tensor(f"{_DONE_FLAGS}_batch"), eng.ring_cursor,
                            outputs)
        if not logging_flag:
            return {}
        s = sums.tolist()
        values, j_values, returns = outputs
        # the ring in slot order: the metrics are means / extremes / spreads over all of it
        return self.trainers[policy].loss_metrics(
            -s[1] / fused.rows, s[0] / fused.rows, rewards, actions, values, j_values, returns)

    # ------------------------------------------------------------------ checkpoints
    def save_model_checkpoint(self, iteration=0):
        if self.device_id != 0:
            return
        freq = self.config["saving"]["model_params_save_freq"]
        if iteration % freq == 0 or iteration == self.num_iters - 1:
            for kind, models in (("actor", self.actor_models), ("critic", self.critic_models)):
                for policy, model in models.items():
                    path = os.path.join(
                        self.save_dir,
                        f"{policy}_{kind}_{self.current_timestep[policy]}.state_dict")
                    if self.verbose:
                        verbose_print(f"Saving the '{policy}' ({kind}) torch model to the "
                                      f"file: '{path}'.", self.device_id)
                    torch.save(model.state_dict(), path)

    def load_model_checkpoint(self, ckpts_dict=None):
        if ckpts_dict is None:
            ckpts_dict = {}
            for p in self.policies:
                model_cfg = self.config["policy"][p]["model"]
                ckpts_dict[p] = model_cfg.get("model_ckpt_filepath", "") if isinstance(
                    model_cfg, dict) else ""
        for policy, paths in ckpts_dict.items():
            assert policy in self.policies
            if not (isinstance(paths, dict) and paths.get("actor") and paths.get("critic")):
                continue
            assert os.path.isfile(paths["actor"]), "Invalid actor model checkpoint path!"
            assert os.path.isfile(paths["critic"]), "Invalid critic model checkpoint path!"
            steps = [int(os.path.basename(paths[k]).split(".state_dict")[0].split("_")[-1])
                     for k in ("actor", "critic")]
            assert steps[0] == steps[1], (
                "The timestep is different between the actor model and the critic model ")
            self.actor_models[policy].load_state_dict(torch.load(paths["actor"], map_location="cpu"))
            self.critic_models[policy].load_state_dict(torch.load(paths["critic"], map_location="cpu"))
            hard_update(self.target_actor_models[policy], self.actor_models[policy])
            hard_update(self.target_critic_models[policy], self.critic_models[policy])
            self.current_timestep[policy] = steps[0]
