"""Trainer: device-resident rollouts + A2C / PPO updates.

Public surface of the reference's TrainerBase / TrainerA2C
(warp_drive/training/trainers/trainer_base.py:69-846, trainer_a2c.py:43-384): same
constructor arguments, same YAML run-config schema merged over default_configs.yaml, same
`train / save_model_checkpoint / load_model_checkpoint / fetch_episode_states /
graceful_close`, same `{policy}_{timestep}.state_dict` checkpoints and JSON-lines metrics.

What is different underneath
  * rollouts go through RolloutEngine: one libwdb200 launch per timestep for
    TagContinuous (fused sample+step+push+reset), CUDA-graph replay of the whole T-step
    rollout, no host synchronisation inside a rollout;
  * multi-GPU is one process per GPU with a NCCL process group; every iteration issues
    ONE flat all-reduce over the gradients of all trained policies (the reference wraps
    each model in DDP over a gloo group: trainer_a2c.py:137-146, process_group_torch.py:7).
"""
import json
import logging
import os
import random
import time

import numpy as np
import torch
import yaml
from torch import nn

from warp_drive_b200.managers.function_manager import CUDALogController, CUDASampler
from warp_drive_b200.training import obs_norm, reward_scale
from warp_drive_b200.training.algorithms.policygradient import A2C, PPO
from warp_drive_b200.training.models.fully_connected import ModelFactory
from warp_drive_b200.training.rollout import RolloutEngine
from warp_drive_b200.training.utils.data_loader import (
    create_and_push_data_placeholders, validate_policy_map)
from warp_drive_b200.training.utils.flat_adam import FlatAdam
from warp_drive_b200.training.utils.param_scheduler import ParamScheduler
from warp_drive_b200.utils.constants import Constants

_ACTIONS = Constants.ACTIONS
_REWARDS = Constants.REWARDS
_DONE_FLAGS = Constants.DONE_FLAGS
_PROCESSED_OBSERVATIONS = Constants.PROCESSED_OBSERVATIONS
_ACTION_MASK = Constants.ACTION_MASK
_EPSILON = 1e-10
_CONFIG_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "run_configs")


def recursive_merge_config_dicts(config, default_config):
    """Fill every key missing from `config` with the default (trainer_base.py:46-60)."""
    assert isinstance(config, dict) and isinstance(default_config, dict)
    for k, v in default_config.items():
        if k not in config:
            config[k] = v
        elif isinstance(v, dict) and isinstance(config[k], dict):
            recursive_merge_config_dicts(config[k], v)
    return config


def load_run_config(name_or_path):
    path = name_or_path if os.path.exists(name_or_path) else os.path.join(
        _CONFIG_DIR, f"{name_or_path}.yaml")
    with open(path, "r", encoding="utf8") as fp:
        return yaml.safe_load(fp)


def verbose_print(message, device_id=0):
    print(f"[Device {device_id or 0}]: {message} ")


class PerfStats:
    """Timing of the rollout / training phases with CUDA events; `steps` counts env-steps
    like the reference (iters x train_batch_size, trainer_base.py:374) and
    `agent_steps` additionally multiplies by the number of agents."""

    def __init__(self):
        self.iters = 0
        self.steps = 0
        self.agent_steps = 0
        self.rollout_time = 0.0
        self.training_time = 0.0
        self.total_time = 0.0

    def get_perf_stats(self):
        it = max(self.iters, 1)
        tot = max(self.total_time, 1e-12)
        return {
            "Mean rollout time per iter (ms)": 1000 * self.rollout_time / it,
            "Mean training time per iter (ms)": 1000 * self.training_time / it,
            "Mean total time per iter (ms)": 1000 * self.total_time / it,
            "Mean steps per sec (rollout)": self.steps / max(self.rollout_time, 1e-12),
            "Mean steps per sec (training time)": self.steps / max(self.training_time, 1e-12),
            "Mean steps per sec (total)": self.steps / tot,
            "Mean agent-steps per sec (total)": self.agent_steps / tot,
        }


class Trainer:
    def __init__(self, env_wrapper=None, config=None, policy_tag_to_agent_id_map=None,
                 create_separate_placeholders_for_each_policy=False,
                 obs_dim_corresponding_to_num_agents="first", num_devices=1, device_id=0,
                 results_dir=None, verbose=True, use_cuda_graph=True):
        assert env_wrapper is not None and env_wrapper.env_backend != "cpu"
        assert config is not None
        self._check_obs_dim(obs_dim_corresponding_to_num_agents)
        # heterogeneous agents: each policy steps through its own observation / action /
        # reward arrays, and / or the env writes observations agent-last ([E, *F, N])
        self.create_separate_placeholders_for_each_policy = bool(
            create_separate_placeholders_for_each_policy)
        self.obs_dim_corresponding_to_num_agents = obs_dim_corresponding_to_num_agents
        self.cuda_envs = env_wrapper
        self.verbose = verbose
        self.num_devices, self.device_id = num_devices, device_id

        with open(os.path.join(_CONFIG_DIR, "default_configs.yaml"), encoding="utf8") as fp:
            default = yaml.safe_load(fp)
        self.config = config
        config["trainer"] = recursive_merge_config_dicts(config["trainer"], default["trainer"])
        for key in config["policy"]:
            self._merge_policy_defaults(config["policy"][key], default["policy"])
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
        reward_scaling = {p: reward_scale.reward_scale_settings(config["policy"][p], p)
                          for p in self.policies}

        t = config["trainer"]
        self.num_episodes = t["num_episodes"]
        self.training_batch_size = t["train_batch_size"]
        self.num_envs = t["num_envs"]
        assert self.num_envs == env_wrapper.n_envs
        self.training_batch_size_per_env = self.training_batch_size // self.num_envs
        assert self.training_batch_size_per_env > 0
        batch_slots_per_env = self._batch_slots_per_env(t)

        # first reset pushes every array to HBM
        self.cuda_envs.reset_all_envs()
        self.cuda_sample_controller = CUDASampler(self.cuda_envs.cuda_function_manager)
        create_and_push_data_placeholders(
            env_wrapper=self.cuda_envs, action_sampler=self.cuda_sample_controller,
            policy_tag_to_agent_id_map=self.policy_tag_to_agent_id_map,
            create_separate_placeholders_for_each_policy=(
                self.create_separate_placeholders_for_each_policy),
            obs_dim_corresponding_to_num_agents=obs_dim_corresponding_to_num_agents,
            training_batch_size_per_env=batch_slots_per_env)
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

        self.trainers = {}
        self.clip_grad_norm, self.max_grad_norm, self.current_timestep = {}, {}, {}
        self._create_network_dicts()
        for policy in self.policies:
            self.current_timestep[policy] = 0
            self._initialize_policy_model(policy)
            if reward_scaling[policy][0]:
                reward_scale.register_buffers(self.models[policy])
        self.load_model_checkpoint()
        for policy in self.policies:
            for model in self._all_networks(policy):
                model.cuda()
        # ONE flat float32 arena for the parameters and one for the gradients of every trained
        # network: Adam / clipping run as flat kernels (utils/flat_adam.py) and the multi-GPU
        # gradient all-reduce is a single in-place NCCL call on `_arena_grads`
        nets = [m for p in self.policies for m in self._trained_networks(p)]
        total = sum(FlatAdam.numel(m.parameters()) for m in nets)
        dev = next(nets[0].parameters()).device
        self._arena_params = torch.zeros(total, dtype=torch.float32, device=dev)
        self._arena_grads = torch.zeros(total, dtype=torch.float32, device=dev)
        self._arena_off = 0
        for policy in self.policies:
            self._initialize_optimizer(policy)
        for policy in self.policies_to_train:
            self._initialize_policy_algorithm(policy)
        self._minibatch_steps = self._minibatch_schedule()
        # running reward scaling (training/reward_scale.py) of the trained policies with the key
        self._reward_scalers = {}
        for policy in self.policies_to_train:
            on, clip = reward_scaling[policy]
            if on:
                r = self.cuda_envs.cuda_data_manager.data_on_device_via_torch(
                    f"{_REWARDS}_batch_{policy}")
                self._reward_scalers[policy] = reward_scale.RewardScaler(
                    self.models[policy], tuple(r.shape), config["policy"][policy]["gamma"],
                    clip, r.device)
        if self.num_devices > 1:
            self._broadcast_parameters()
        self.engine = self._make_engine(use_cuda_graph)
        self._perm_generator = None
        self.perf_stats = PerfStats()

    # ------------------------------------------------------------------ what subclasses change
    @staticmethod
    def _check_obs_dim(obs_dim_corresponding_to_num_agents):
        assert obs_dim_corresponding_to_num_agents in ("first", "last"), (
            "obs_dim_corresponding_to_num_agents must be 'first' ([E, N, *F] observations) or "
            "'last' ([E, *F, N])")

    @staticmethod
    def _merge_policy_defaults(policy_config, defaults):
        recursive_merge_config_dicts(policy_config, defaults)

    def _batch_slots_per_env(self, trainer_config):
        """Timesteps per env that the `*_batch*` arrays hold."""
        return self.training_batch_size_per_env

    def _create_network_dicts(self):
        self.models, self.optimizers, self.lr_schedules = {}, {}, {}

    def _initialize_policy_model(self, policy):
        self.models[policy] = self._build_model(
            policy, self._get_config(["policy", policy, "model"]))

    def _trained_networks(self, policy):
        """The networks of `policy` that an optimizer updates, in arena order."""
        return [self.models[policy]]

    def _all_networks(self, policy):
        """Every network of `policy`: moved to the GPU and broadcast from rank 0."""
        return self._trained_networks(policy)

    def _initialize_optimizer(self, policy):
        self.lr_schedules[policy] = ParamScheduler(self._get_config(["policy", policy, "lr"]))
        self.optimizers[policy] = self._flat_adam(
            self.models[policy],
            self.lr_schedules[policy].get_param_value(self.current_timestep[policy]))

    def _optimizers_of(self, policy):
        """(metric-key suffix, FlatAdam, lr schedule) of each network `policy` trains."""
        return [("", self.optimizers[policy], self.lr_schedules[policy])]

    def _make_engine(self, use_cuda_graph):
        return RolloutEngine(
            self.cuda_envs, self.models, self.policy_tag_to_agent_id_map,
            self.cuda_sample_controller, self.training_batch_size_per_env,
            use_cuda_graph=use_cuda_graph,
            create_separate_placeholders_for_each_policy=(
                self.create_separate_placeholders_for_each_policy),
            obs_dim_corresponding_to_num_agents=self.obs_dim_corresponding_to_num_agents)

    # ------------------------------------------------------------------ setup helpers
    def _get_config(self, args):
        cfg = self.config
        for a in args:
            cfg = cfg[a]
        return cfg

    def _build_model(self, policy, model_config):
        cls = ModelFactory.create(model_config["type"])
        algorithm = self.config["policy"][policy].get("algorithm")
        if getattr(cls, "is_recurrent", False) and algorithm not in ("A2C", "PPO"):
            raise ValueError(f"policy {policy!r}: a recurrent model ({model_config['type']}) "
                             f"trains with A2C or PPO, not {algorithm}")
        model = cls(
            env=self.cuda_envs, model_config=model_config, policy=policy,
            policy_tag_to_agent_id_map=self.policy_tag_to_agent_id_map,
            create_separate_placeholders_for_each_policy=(
                self.create_separate_placeholders_for_each_policy),
            obs_dim_corresponding_to_num_agents=self.obs_dim_corresponding_to_num_agents)
        if model_config.get("init_method") == "xavier":
            for m in model.modules():
                if isinstance(m, nn.Linear):
                    nn.init.xavier_uniform_(m.weight)
        return model

    def _flat_adam(self, model, lr):
        """FlatAdam over `model` on the next slice of the parameter / gradient arena."""
        n = FlatAdam.numel(model.parameters())
        lo = self._arena_off
        self._arena_off += n
        return FlatAdam(model.parameters(), lr=lr,
                        arena=(self._arena_params[lo:lo + n], self._arena_grads[lo:lo + n]))

    def _initialize_policy_algorithm(self, policy):
        c = self._get_config(["policy", policy])
        assert c["algorithm"] in ("A2C", "PPO")
        self.clip_grad_norm[policy] = c["clip_grad_norm"]
        if c["clip_grad_norm"]:
            self.max_grad_norm[policy] = c["max_grad_norm"]
        kw = dict(discount_factor_gamma=c["gamma"], normalize_advantage=c["normalize_advantage"],
                  normalize_return=c["normalize_return"], vf_loss_coeff=c["vf_loss_coeff"],
                  entropy_coeff=c["entropy_coeff"])
        # several epochs over shuffled minibatches / GAE (absent keys: the single-step update)
        kw.update(num_epochs=c.get("num_epochs", 1), num_mini_batches=c.get("num_mini_batches", 1),
                  gae_lambda=c.get("gae_lambda"))
        self.trainers[policy] = A2C(**kw) if c["algorithm"] == "A2C" else PPO(
            clip_param=c["clip_param"], **kw)
        if (self.trainers[policy].minibatch_path
                and self.config["trainer"].get("neg_pos_env_ratio", -1) > 0):
            raise ValueError("neg_pos_env_ratio is not supported with num_epochs, "
                             "num_mini_batches or gae_lambda")

    def _minibatch_schedule(self):
        """Optimizer steps per iteration (num_epochs x num_mini_batches) when the trained
        policies take the minibatch update, None when they all take the single-step update.
        Every optimizer step all-reduces the whole gradient arena once, so the policies must
        agree on that product; each still runs its own epochs and minibatch split."""
        on = {p: getattr(self.trainers.get(p), "minibatch_path", False)
              for p in self.policies_to_train}
        if not any(on.values()):
            return None
        if not all(on.values()):
            raise ValueError("either every trained policy sets num_epochs / num_mini_batches / "
                             f"gae_lambda or none does: {on}")
        steps = {p: (self.trainers[p].num_epochs, self.trainers[p].num_mini_batches)
                 for p in self.policies_to_train}
        if len({e * m for e, m in steps.values()}) != 1:
            raise ValueError("the trained policies must agree on num_epochs x num_mini_batches: "
                             f"{steps}")
        e, m = next(iter(steps.values()))
        return e * m

    # ------------------------------------------------------------------ multi-GPU
    def _trained_params(self):
        return [p for pol in self.policies_to_train for m in self._trained_networks(pol)
                for p in m.parameters()]

    def _broadcast_parameters(self):
        import torch.distributed as dist

        for pol in self.policies:
            for m in self._all_networks(pol):
                for p in m.parameters():
                    dist.broadcast(p.data, src=0)

    def _allreduce_gradients(self):
        """ONE NCCL all-reduce (mean) over the gradients of every policy, in place on the flat
        gradient arena (every .grad is a view into it: no packing, no copies back)."""
        import torch.distributed as dist

        dist.all_reduce(self._arena_grads, op=dist.ReduceOp.SUM)
        self._arena_grads.div_(self.num_devices)

    # ------------------------------------------------------------------ training loop
    def train(self):
        self._reset_all_envs()
        self.engine.resync_observations()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        n_agents = self.cuda_envs.n_agents
        for iteration in range(self.num_iters):
            t0 = time.time()
            ev[0].record()
            self._generate_rollout_batch()
            ev[1].record()
            metrics = self._update_model_params(iteration)
            ev[2].record()
            torch.cuda.synchronize()
            self.perf_stats.rollout_time += ev[0].elapsed_time(ev[1]) / 1000
            self.perf_stats.training_time += ev[1].elapsed_time(ev[2]) / 1000
            self.perf_stats.iters = iteration + 1
            self.perf_stats.steps = self.perf_stats.iters * self.training_batch_size
            self.perf_stats.agent_steps = self.perf_stats.steps * n_agents
            self.perf_stats.total_time += time.time() - t0
            self._log_metrics(metrics)
            self.save_model_checkpoint(iteration)

    def _get_sample_params(self):
        t = self.current_timestep[self.policies[0]]
        return {k: s.get_param_value(t) for k, s in self.sample_params_schedules.items()}

    def _generate_rollout_batch(self):
        params = self._get_sample_params()
        self.engine.rollout(**params)
        return params

    def _update_model_params(self, iteration):
        if self._minibatch_steps is not None:
            return self._update_model_params_minibatches(iteration)
        logging_flag = self._is_logging_iteration(iteration)
        dm = self.cuda_envs.cuda_data_manager
        done_flags_batch = dm.data_on_device_via_torch(f"{_DONE_FLAGS}_batch")
        training_rewards = self._training_rewards(done_flags_batch)
        loss_metrics = {}
        for policy in self.policies_to_train:
            actions = dm.data_on_device_via_torch(f"{_ACTIONS}_batch_{policy}")
            rewards = training_rewards[policy]
            obs = dm.data_on_device_via_torch(f"{_PROCESSED_OBSERVATIONS}_batch_{policy}")
            # every timestep of the batch is trained under its own action mask (the reference
            # applies the mask of the rollout's last step to all of them)
            mask_name = f"{_ACTION_MASK}_batch_{policy}"
            kw = ({"action_mask": dm.data_on_device_via_torch(mask_name)}
                  if dm.is_data_on_device_via_torch(mask_name) else {})
            if getattr(self.models[policy], "is_recurrent", False):
                # the whole batch as T steps of every sequence, from the state it started from
                probs, values = self.models[policy].forward_sequence(
                    obs, self.engine.hidden_start[policy], done_flags_batch)
            else:
                probs, values = self.models[policy](obs=obs, **kw)
            self._advance_timestep(policy)
            # a Gaussian policy trains on its float actions under its log_std
            if getattr(self.models[policy], "is_gaussian", False):
                kw = {"log_std": self.models[policy].log_std}
            else:
                actions, kw = actions.long(), {}
            loss, loss_metrics[policy] = self.trainers[policy].compute_loss_and_metrics(
                self.current_timestep[policy], actions, rewards, done_flags_batch,
                probs, values, perform_logging=logging_flag,
                negative_positive_ratio=self.config["trainer"].get("neg_pos_env_ratio", -1),
                **kw)
            self.optimizers[policy].zero_grad()
            loss.backward()
        return self._step_optimizers(loss_metrics, logging_flag)

    def _update_model_params_minibatches(self, iteration):
        """num_epochs x num_mini_batches optimizer steps on one batch: the batch is prepared
        once per policy (advantages, value targets and old log-probs at the rollout's
        parameters), then every step is forward + fused loss + backward for every policy, one
        all-reduce and clipping + Adam.  Step s of a policy with m minibatches is chunk s % m of
        its epoch s // m; each epoch draws a fresh permutation of that policy's rows.  The bf16
        rollout weights are repacked once, after the last step."""
        logging_flag = self._is_logging_iteration(iteration)
        dm = self.cuda_envs.cuda_data_manager
        done_flags_batch = dm.data_on_device_via_torch(f"{_DONE_FLAGS}_batch")
        training_rewards = self._training_rewards(done_flags_batch)
        batches = {}
        for policy in self.policies_to_train:
            mask_name = f"{_ACTION_MASK}_batch_{policy}"
            mask = (dm.data_on_device_via_torch(mask_name)
                    if dm.is_data_on_device_via_torch(mask_name) else None)
            self._advance_timestep(policy)
            # a recurrent policy replays its sequences from the state its batch started from
            kw = ({"hidden_start": self.engine.hidden_start[policy]}
                  if policy in self.engine.hidden_start else {})
            batches[policy] = self.trainers[policy].prepare_batch(
                self.models[policy],
                dm.data_on_device_via_torch(f"{_PROCESSED_OBSERVATIONS}_batch_{policy}"),
                dm.data_on_device_via_torch(f"{_ACTIONS}_batch_{policy}"),
                training_rewards[policy], done_flags_batch, mask, **kw)
        if self._perm_generator is None:
            self._perm_generator = torch.Generator(device=done_flags_batch.device)
            self._perm_generator.manual_seed(self.seed)
        n_steps = self._minibatch_steps
        sums = {p: torch.zeros(5, dtype=torch.float64, device=done_flags_batch.device)
                for p in self.policies_to_train}
        chunks = {}
        step_info = None
        for step in range(n_steps):
            for policy in self.policies_to_train:
                n_mini = self.trainers[policy].num_mini_batches
                if step % n_mini == 0:         # a new epoch of this policy
                    chunks[policy] = torch.tensor_split(
                        self.minibatch_permutation(batches[policy].units), n_mini)
                rows = chunks[policy][step % n_mini]
                loss, s = self.trainers[policy].minibatch_loss(
                    self.models[policy], batches[policy], rows, self.current_timestep[policy])
                self.optimizers[policy].zero_grad()
                loss.backward()
                if logging_flag:
                    sums[policy] += s / (rows.numel() * batches[policy].rows_per_unit)
            info = self._optimizer_step(self.policies_to_train, logging_flag)
            step_info = info if step_info is None else self._add_step_info(step_info, info)
        loss_metrics = {}
        if logging_flag:
            for policy, (norms, lrs) in step_info.items():
                norms.update({k: v / n_steps for k, v in norms.items()})
            for policy in self.policies_to_train:
                loss_metrics[policy] = self.trainers[policy].minibatch_metrics(
                    batches[policy], sums[policy] / n_steps, self.current_timestep[policy])
        return self._finish_update(loss_metrics, step_info, logging_flag)

    def _training_rewards(self, done_flags_batch):
        """{trained policy: the rewards batch its update reads}: the data manager's own
        `rewards_batch_{p}`, or for a policy with scale_rewards its scaled copy, made here from
        the raw batch after the rollout and before any update work (training/reward_scale.py)."""
        dm = self.cuda_envs.cuda_data_manager
        out = {}
        for policy in self.policies_to_train:
            rewards = dm.data_on_device_via_torch(f"{_REWARDS}_batch_{policy}")
            scaler = self._reward_scalers.get(policy)
            out[policy] = (rewards if scaler is None
                           else scaler.scale(rewards, done_flags_batch, self.num_devices))
        return out

    def minibatch_permutation(self, n_rows):
        """The next epoch's order of a policy's n_rows batch rows (int32, on the device), drawn
        from the trainer's seeded generator: a run is reproducible."""
        return torch.randperm(n_rows, generator=self._perm_generator,
                              device=self._perm_generator.device).to(torch.int32)

    @staticmethod
    def _add_step_info(total, info):
        for policy, (norms, _) in info.items():
            for k, v in norms.items():
                total[policy][0][k] = total[policy][0][k] + v
        return total

    def _is_logging_iteration(self, iteration):
        return (iteration % self.config["saving"]["metrics_log_freq"] == 0
                or iteration == self.num_iters - 1)

    def _advance_timestep(self, policy):
        """Count one training batch for `policy` and set its learning rates for that step."""
        self.current_timestep[policy] += self.training_batch_size
        for _, optimizer, schedule in self._optimizers_of(policy):
            optimizer.param_groups[0]["lr"] = schedule.get_param_value(
                self.current_timestep[policy])

    def _step_optimizers(self, loss_metrics, logging_flag):
        """The update once the gradients of the policies in `loss_metrics` are in the arena:
        one all-reduce, then clipping + Adam per network.  On a logging iteration, returns the
        metrics of every trained policy and restarts the episodic counters."""
        step_info = self._optimizer_step(loss_metrics, logging_flag)
        return self._finish_update(loss_metrics, step_info, logging_flag)

    def _optimizer_step(self, stepped, logging_flag):
        """One optimizer step of the policies in `stepped`: one all-reduce of the gradient
        arena, then clipping + Adam per network.  Returns {policy: (gradient norms as device
        tensors, learning rates)}, filled on a logging iteration."""
        if self.num_devices > 1 and stepped:
            self._allreduce_gradients()
        step_info = {}
        for policy in self.policies_to_train:
            optimizers = self._optimizers_of(policy) if policy in stepped else []
            norms, lrs = {}, {}
            if logging_flag:
                for suffix, opt, _ in optimizers:
                    norms[f"Gradient norm{suffix}"] = sum(
                        p.grad.norm(2) for p in opt.param_list if p.grad is not None)
                    lrs[f"Learning rate{suffix}"] = opt.param_groups[0]["lr"]
            # clip_grad_norm_ + Adam as two flat kernels, clip factor stays on the device
            clip = self.max_grad_norm[policy] if self.clip_grad_norm[policy] else None
            for _, opt, _ in optimizers:
                opt.step(max_grad_norm=clip)
            step_info[policy] = (norms, lrs)
        return step_info

    def _finish_update(self, loss_metrics, step_info, logging_flag):
        """Once per iteration after the last optimizer step: repack the rollout weights and, on
        a logging iteration, collect every trained policy's metrics and restart the episodic
        counters."""
        metrics_dict = {}
        for policy in self.policies_to_train:
            if logging_flag:
                norms, lrs = step_info[policy]
                n_done = int(self.engine.num_completed_episodes)
                metrics = loss_metrics.get(policy, {})
                metrics["Current timestep"] = self.current_timestep[policy]
                if policy in self._reward_scalers:
                    metrics["Reward scale"] = float(self.models[policy].return_scale)
                metrics.update({k: float(v) for k, v in norms.items()})
                metrics.update(lrs)
                metrics.update({
                    "Mean episodic reward":
                        float(self.engine.episodic_reward_sum[policy]) / (n_done + _EPSILON),
                    "Mean episodic steps":
                        float(self.engine.episodic_step_sum) / (n_done + _EPSILON)})
                metrics_dict[policy] = metrics
        self.engine.refresh_forward_weights()
        self._update_observation_statistics()
        if logging_flag:
            for policy in self.policies:
                self.engine.episodic_reward_sum[policy].zero_()
            self.engine.episodic_step_sum.zero_()
            self.engine.num_completed_episodes.zero_()
        return metrics_dict

    def _update_observation_statistics(self):
        """Merge this iteration's raw observation batch into the running statistics of every
        trained policy that normalizes its observations (training/obs_norm.py): after the last
        optimizer step, so the next rollout and update see the new statistics."""
        dm = self.cuda_envs.cuda_data_manager
        for policy in self.policies_to_train:
            model = self.models[policy]
            if getattr(model, "normalize_observations", False):
                obs = dm.data_on_device_via_torch(f"{_PROCESSED_OBSERVATIONS}_batch_{policy}")
                obs_norm.update_moments(model, obs, self.num_devices)

    def _reset_all_envs(self):
        """Restart every env; the running returns of reward scaling and the recurrent policies'
        states restart with them."""
        self.cuda_envs.reset_all_envs()
        if getattr(self, "engine", None) is not None:
            self.engine.zero_hidden()
        for scaler in self._reward_scalers.values():
            scaler.reset()

    # ------------------------------------------------------------------ logging / ckpt
    def _log_metrics(self, metrics):
        if not metrics:
            return
        perf = self.perf_stats.get_perf_stats()
        if self.verbose:
            print("\n" + "=" * 40)
            print(f"Device: {self.device_id}")
            print(f"{'Iterations Completed':40}: {self.perf_stats.iters} / {self.num_iters}")
            for k, v in perf.items():
                print(f"{k:40}: {v:10.2f}")
            for policy, m in metrics.items():
                print("=" * 40 + f"\nMetrics for policy '{policy}'\n" + "=" * 40)
                for k, v in m.items():
                    print(f"{k:40}: {v:10.5f}" if isinstance(v, float) else f"{k:40}: {v}")
            print("=" * 40 + "\n")
        logs = {"Iterations Completed": self.perf_stats.iters}
        logs.update(metrics)
        logs["Perf. Stats"] = perf
        fn = f"results_device_{self.device_id}.json" if self.num_devices > 1 else "results.json"
        with open(os.path.join(self.save_dir, fn), "a+", encoding="utf8") as fp:
            json.dump(logs, fp)
            fp.write("\n")

    def save_model_checkpoint(self, iteration=0):
        if self.device_id != 0:
            return
        freq = self.config["saving"]["model_params_save_freq"]
        if iteration % freq == 0 or iteration == self.num_iters - 1:
            for policy, name, model in self._checkpointed_networks():
                path = os.path.join(
                    self.save_dir, f"{name}_{self.current_timestep[policy]}.state_dict")
                if self.verbose:
                    verbose_print(f"Saving the '{name}' torch model to the file: '{path}'.",
                                  self.device_id)
                torch.save(model.state_dict(), path)

    def _checkpointed_networks(self):
        """(policy, file name prefix, network) of every network a checkpoint saves."""
        return [(policy, policy, model) for policy, model in self.models.items()]

    @staticmethod
    def _checkpoint_timestep(path):
        """The timestep encoded in a checkpoint's file name ({prefix}_{timestep}.state_dict)."""
        return int(os.path.basename(path).split(".state_dict")[0].split("_")[-1])

    def load_model_checkpoint(self, ckpts_dict=None):
        if ckpts_dict is None:
            ckpts_dict = {p: self.config["policy"][p]["model"].get("model_ckpt_filepath", "")
                          for p in self.policies}
        for policy, path in ckpts_dict.items():
            assert policy in self.policies
            self._load_policy_checkpoint(policy, path)
        # the tensor-core rollout forward keeps its own packed bf16 copy of the weights
        if getattr(self, "engine", None) is not None:
            self.engine.refresh_forward_weights()

    def _load_policy_checkpoint(self, policy, path):
        if path:
            assert os.path.isfile(path), "Invalid model checkpoint path!"
            self.models[policy].load_state_dict(torch.load(path, map_location="cpu"))
            self.current_timestep[policy] = self._checkpoint_timestep(path)

    def graceful_close(self):
        self.cuda_sample_controller = None
        if self.verbose:
            verbose_print("Trainer exits gracefully", self.device_id)

    # ------------------------------------------------------------------ evaluation
    def evaluate_episodes(self, **sample_params):
        """Play one episode in every env replica with the current actor (scale=0: no
        exploration noise; for categorical policies pass nothing; use_argmax=True: the
        deterministic action of a categorical or Gaussian policy) and return per-env reward /
        step sums (trainer_base.py:794-846); accumulated on the device, no per-step host
        transfer.  The env states are restarted afterwards."""
        eng = self.engine
        dm = self.cuda_envs.cuda_data_manager
        fused, eng.fused = eng.fused, None     # generic multi-launch step while evaluating
        dev = dm.device
        reward_sum = {p: torch.zeros((self.num_envs, len(ids)), device=dev)
                      for p, ids in self.policy_tag_to_agent_id_map.items()}
        step_sum = {p: torch.zeros(self.num_envs, dtype=torch.int32, device=dev)
                    for p in self.policies}
        self._reset_all_envs()
        done = dm.data_on_device_via_torch("_done_")
        with torch.no_grad():
            for _ in range(self.cuda_envs.episode_length):
                probs = eng.evaluate_policies(-1)
                eng.sample_actions(probs, -1, **sample_params)
                self.cuda_envs.step_all_envs()
                undone = done == 0
                for p in self.policies:
                    r_p, _ = eng.policy_step_arrays(p)
                    reward_sum[p] += r_p * undone[:, None]
                    step_sum[p] += undone.to(torch.int32)
                if eng.recurrent:
                    eng.recurrent_reset_done()
                # done envs restart but keep their flag: one episode per env is counted
                self.cuda_envs.reset_only_done_envs(undo_done_after_reset=False)
        eng.fused = fused
        self._reset_all_envs()
        eng.resync_observations()
        return reward_sum, step_sum

    # ------------------------------------------------------------------ episode states
    def fetch_episode_states(self, list_of_states=None, env_id=0, include_rewards_actions=False,
                             include_probabilities=False, policy=""):
        """Play one episode of env `env_id` with the current policies and return the
        per-timestep values of the requested device arrays (trainer_base.py:689-792).
        With separate placeholders, `policy` names the policy whose `sampled_actions_{policy}`
        / `rewards_{policy}` (include_rewards_actions) and probabilities
        (include_probabilities) are logged.

        The episode is logged ON THE DEVICE: every requested array has a [T + 1, ...] ring in
        HBM that `wdb_log_one_step` (the CUDALogController kernel, function_manager.py:295-422)
        fills with env `env_id`'s slice after each step, the done flag of that env is logged
        the same way, and the host pulls everything ONCE after the last step (the reference
        pulls every whole [E, ...] array to the host every timestep)."""
        from warp_drive_b200.managers.function_manager import CUDALogController

        assert 0 <= env_id < self.num_envs
        assert isinstance(list_of_states, list) and list_of_states
        dm = self.cuda_envs.cuda_data_manager
        self._reset_all_envs()
        self.engine.resync_observations()
        T = self.cuda_envs.episode_length
        logger = CUDALogController(self.cuda_envs.cuda_function_manager)

        def ring(name, steps):
            t = dm.data_on_device_via_torch(name)
            fill = float("nan") if t.dtype.is_floating_point else 0
            return torch.full((steps,) + tuple(t.shape[1:]), fill, dtype=t.dtype, device=t.device)

        rings = {name: ring(name, T + 1) for name in list_of_states}
        for name in list_of_states:
            logger.log_tensor_one_step(rings[name], dm.data_on_device_via_torch(name), 0, env_id)
        suffix = f"_{policy}" if policy else ""
        if self.create_separate_placeholders_for_each_policy and (
                include_rewards_actions or include_probabilities):
            assert policy in self.policies, (
                "with separate placeholders, name the policy whose actions, rewards or "
                "probabilities to log")
        extra = {}
        if include_rewards_actions:
            extra = {name: ring(name, T) for name in (_ACTIONS + suffix, _REWARDS + suffix)}
        done_ring = torch.zeros(T, dtype=torch.int32, device=dm.device)
        prob_rings = None
        fused, self.engine.fused = self.engine.fused, None
        sa, self.engine.sa = self.engine.sa, None
        try:
            for t in range(T):
                with torch.no_grad():
                    probs = self.engine.evaluate_policies(-1)
                    self.engine.sample_actions(probs, -1)
                    self.cuda_envs.step_all_envs()
                    if self.engine.recurrent:
                        self.engine.recurrent_reset_done()
                for name in list_of_states:
                    logger.log_tensor_one_step(rings[name], dm.data_on_device_via_torch(name),
                                               t + 1, env_id)
                for name, r in extra.items():
                    logger.log_tensor_one_step(r, dm.data_on_device_via_torch(name), t, env_id)
                logger.log_tensor_one_step(done_ring, dm.data_on_device_via_torch("_done_"), t,
                                           env_id)
                if include_probabilities:
                    # (a Gaussian policy logs its mean; several Gaussian policies sharing the
                    #  placeholders come per policy as well)
                    if isinstance(probs, dict):
                        probs = probs[policy]
                    if prob_rings is None:
                        prob_rings = [torch.zeros((T,) + tuple(p.shape[1:]), device=p.device)
                                      for p in probs]
                    for r, p in zip(prob_rings, probs):
                        logger.log_tensor_one_step(r, p.contiguous(), t, env_id)
            # ---- the one device -> host transfer of the episode
            done_host = done_ring.cpu().numpy()
            ended = np.nonzero(done_host)[0]
            n_steps = int(ended[0]) + 1 if len(ended) else T
            out = {name: rings[name][: n_steps + 1].cpu().numpy().astype(np.float32)
                   for name in list_of_states}
            for name, r in extra.items():
                out[name] = r[:n_steps].cpu().numpy().astype(np.float32)
            if include_probabilities:
                host = [r[:n_steps].cpu().numpy() for r in prob_rings]
                out["probabilities"] = [[h[t] for h in host] for t in range(n_steps)]
        finally:
            self.engine.fused = fused
            self.engine.sa = sa
            self._reset_all_envs()
            self.engine.resync_observations()
        return out

    def _fetch_episode_states_host_pull(self, list_of_states=None, env_id=0, include_rewards_actions=False,
                             include_probabilities=False):
        """The reference-shaped implementation (one host pull of every whole [E, ...] array
        per timestep, trainer_base.py:689-792); kept as the checker of fetch_episode_states."""
        assert 0 <= env_id < self.num_envs
        assert isinstance(list_of_states, list) and list_of_states
        dm = self.cuda_envs.cuda_data_manager
        self._reset_all_envs()
        self.engine.resync_observations()
        T = self.cuda_envs.episode_length
        out = {}
        for name in list_of_states:
            shape = dm.get_shape(name)
            out[name] = np.full((T + 1,) + tuple(shape[1:]), np.nan, dtype=np.float32)
            out[name][0] = dm.pull_data_from_device(name)[env_id]
        if include_rewards_actions:
            out[_ACTIONS] = np.full((T,) + tuple(dm.get_shape(_ACTIONS)[1:]), np.nan, np.float32)
            out[_REWARDS] = np.full((T,) + tuple(dm.get_shape(_REWARDS)[1:]), np.nan, np.float32)
        fused, self.engine.fused = self.engine.fused, None
        try:
            for t in range(T):
                with torch.no_grad():
                    probs = self.engine.evaluate_policies(-1)
                    self.engine.sample_actions(probs, -1)
                    self.cuda_envs.step_all_envs()
                for name in list_of_states:
                    out[name][t + 1] = dm.pull_data_from_device(name)[env_id]
                if include_rewards_actions:
                    out[_ACTIONS][t] = dm.pull_data_from_device(_ACTIONS)[env_id]
                    out[_REWARDS][t] = dm.pull_data_from_device(_REWARDS)[env_id]
                if include_probabilities:
                    out.setdefault("probabilities", []).append(
                        [p[env_id].cpu().numpy() for p in probs])
                if int(dm.pull_data_from_device("_done_")[env_id]):
                    for name in out:
                        if isinstance(out[name], np.ndarray):
                            out[name] = out[name][: t + 2 if name in list_of_states else t + 1]
                    break
        finally:
            self.engine.fused = fused
            self._reset_all_envs()
            self.engine.resync_observations()
        return out


# names a reference user imports
TrainerA2C = Trainer
TrainerBase = Trainer
