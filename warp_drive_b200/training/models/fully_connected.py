"""FullyConnected policy/value network (the only dense contraction on the rollout path).

Same architecture and forward contract as the reference's ModelBaseFullyConnected /
FullyConnected (warp_drive/training/models/model_base.py:28-213,
fully_connected.py:20-89): L x (Linear + ReLU) trunk, one Linear + softmax head per
discrete action component (or a tanh head for Box actions), a scalar value head;
`forward(obs) -> ([probs per head], values)`.  Module / parameter names match the
reference (`fc.{i}.0`, `policy_head.{k}`, `vf_head`) so reference checkpoints
(`{policy}_{timestep}.state_dict`) load unchanged.
"""
import torch
from torch import nn
from torch.nn import functional as func

from warp_drive_b200.training import obs_norm
from warp_drive_b200.training.utils.data_loader import (
    action_head_sizes, get_flattened_obs_size)
from warp_drive_b200.utils.constants import Constants
from warp_drive_b200.utils.spaces import Box, Dict

_OBSERVATIONS = Constants.OBSERVATIONS
_PROCESSED_OBSERVATIONS = Constants.PROCESSED_OBSERVATIONS
_ACTION_MASK = Constants.ACTION_MASK
_LARGE_NEG_NUM = -1e20


def apply_logit_mask(logits, mask=None):
    """mask == 1 marks valid actions; invalid logits get a huge negative offset."""
    if mask is None:
        return logits
    return logits + (1 - mask) * _LARGE_NEG_NUM


class FullyConnected(nn.Module):
    name = "torch_fully_connected"
    normalize_observations = False

    def __init__(self, env, model_config, policy, policy_tag_to_agent_id_map,
                 create_separate_placeholders_for_each_policy=False,
                 obs_dim_corresponding_to_num_agents="first"):
        super().__init__()
        self.env = env
        self.fc_dims = list(model_config["fc_dims"])
        self.action_scale = model_config.get("output_w", 1.0)
        self.action_bias = model_config.get("output_b", 0.0)
        self.policy = policy
        self.policy_tag_to_agent_id_map = policy_tag_to_agent_id_map
        self.create_separate_placeholders_for_each_policy = (
            create_separate_placeholders_for_each_policy)
        assert obs_dim_corresponding_to_num_agents in ("first", "last")
        self.obs_dim_corresponding_to_num_agents = obs_dim_corresponding_to_num_agents
        sample_agent = policy_tag_to_agent_id_map[policy][0]
        self.observation_space = env.env.observation_space[sample_agent]
        self.flattened_obs_size = get_flattened_obs_size(self.observation_space)
        heads, self.is_deterministic = action_head_sizes(env.env.action_space[sample_agent])
        self.flattened_action_size = len(heads)
        dims = [self.flattened_obs_size] + self.fc_dims
        self.fc = nn.ModuleDict({
            str(i): nn.Sequential(nn.Linear(dims[i], dims[i + 1]), nn.ReLU())
            for i in range(len(self.fc_dims))})
        if self.is_deterministic:
            self.output_dims = [len(heads)]
            self.policy_head = nn.Linear(self.fc_dims[-1], len(heads))
        else:
            self.output_dims = list(heads)
            self.policy_head = nn.ModuleList(
                [nn.Linear(self.fc_dims[-1], h) for h in heads])
        self.vf_head = nn.Linear(self.fc_dims[-1], 1)
        self.action_mask = None
        # training-time forward as one fused autograd node (models/fused_mlp_train.py)
        self.use_fused_train_forward = bool(model_config.get("fused_train_forward", True))
        name = f"{_PROCESSED_OBSERVATIONS}_batch_{policy}"
        self.batch_size = env.cuda_data_manager.get_shape(name=name)[0]
        # running observation statistics (training/obs_norm.py): buffers only when the key is
        # on, so the state_dict of a model without it is unchanged
        self.normalize_observations, self.observation_clip = obs_norm.obs_norm_settings(
            model_config, model_config.get("type", "fully_connected"))
        if self.normalize_observations:
            obs_norm.register_buffers(self, self.flattened_obs_size)

    def normalized_input(self, obs):
        """The observations the first layer reads: normalized by the running statistics when
        the model normalizes, else as given."""
        return obs_norm.normalize(self, obs) if self.normalize_observations else obs

    # ---- observation plumbing (model_base.py:93-200)
    def reshape_and_flatten_obs(self, obs):
        num_envs = obs.shape[0]
        if self.create_separate_placeholders_for_each_policy:
            num_agents = len(self.policy_tag_to_agent_id_map[self.policy])
        else:
            num_agents = self.env.n_agents
        if self.obs_dim_corresponding_to_num_agents == "last":
            if obs.dim() == 1:
                obs = obs.reshape(-1, num_agents)
            obs = obs.permute(0, -1, *range(1, obs.dim() - 1))
        return obs.reshape(num_envs, num_agents, -1)

    def get_flattened_obs(self):
        dm = self.env.cuda_data_manager
        prefix = (f"{_OBSERVATIONS}_{self.policy}"
                  if self.create_separate_placeholders_for_each_policy else _OBSERVATIONS)
        if isinstance(self.observation_space, Box):
            flat = self.reshape_and_flatten_obs(dm.data_on_device_via_torch(prefix))
        elif isinstance(self.observation_space, Dict):
            parts = []
            for key in self.observation_space:
                obs = self.reshape_and_flatten_obs(
                    dm.data_on_device_via_torch(f"{prefix}_{key}"))
                if key == _ACTION_MASK:
                    self.action_mask = obs
                    assert obs.shape[-1] == sum(self.output_dims)
                else:
                    parts.append(obs)
            flat = torch.cat(parts, dim=-1)
        else:
            raise NotImplementedError("Observation space must be of Box or Dict type")
        assert flat.shape[-1] == self.flattened_obs_size
        return flat

    def process_one_step_obs(self):
        obs = self.get_flattened_obs()
        if not self.create_separate_placeholders_for_each_policy:
            ids = self.policy_tag_to_agent_id_map[self.policy]
            if len(ids) != obs.shape[1]:
                obs = obs[:, ids]
        return obs

    def push_processed_obs_to_batch(self, batch_index, processed_obs, ring_buffer=None):
        if batch_index < 0:
            return
        assert batch_index < self.batch_size
        name = f"{_PROCESSED_OBSERVATIONS}_batch_{self.policy}"
        if ring_buffer is not None and ring_buffer.has(name):
            ring_buffer.get(name).enqueue(processed_obs)
        else:
            self.env.cuda_data_manager.data_on_device_via_torch(name)[batch_index] = processed_obs

    # ---- forward (fully_connected.py:51-89)
    def forward(self, obs=None, action=None, action_mask=None):
        """action_mask [..., sum of the head sizes] (1 = valid) masks each row with its own
        mask, e.g. every timestep of a training batch with that timestep's; None falls back to
        the mask the last get_flattened_obs() read (the reference's behaviour)."""
        mask = self.action_mask if action_mask is None else action_mask
        if self.use_fused_train_forward and torch.is_grad_enabled() and obs.is_cuda:
            # the update: one autograd node, bias / ReLU / softmax fused around cuBLAS GEMMs
            from warp_drive_b200.training.models import fused_mlp_train

            if fused_mlp_train.supported(self, obs, mask):
                return fused_mlp_train.fused_train_forward(self, obs, mask)
        x = self.normalized_input(obs)
        for i in range(len(self.fc)):
            x = self.fc[str(i)](x)
        if self.is_deterministic:
            out = torch.tanh(apply_logit_mask(self.policy_head(x), mask))
            out = self.action_scale * out + self.action_bias
            probs = ([t.contiguous() for t in torch.split(out, 1, dim=-1)]
                     if self.output_dims[0] > 1 else [out])
        else:
            masks = [None] * len(self.output_dims)
            if mask is not None:
                start = 0
                for k, dim in enumerate(self.output_dims):
                    masks[k] = mask[..., start:start + dim]
                    start += dim
            probs = [func.softmax(apply_logit_mask(head(x), masks[k]), dim=-1)
                     for k, head in enumerate(self.policy_head)]
        vals = self.vf_head(x)[..., 0]
        return probs, vals


class FullyConnectedGaussian(FullyConnected):
    """Diagonal Gaussian policy for Box actions, trained with A2C / PPO: the trunk, value head
    and observation plumbing of FullyConnected; `policy_head` is one Linear(fc_dims[-1], A)
    whose raw output is the mean (no tanh, no scaling) and `log_std` a state-independent
    parameter [A] (model config key `log_std_init`, default 0).  `forward(obs) -> ([mean],
    values)`.  Actions are sampled unclipped (CUDASampler.sample_gaussian); the env bounds
    them."""

    name = "torch_fully_connected_gaussian"
    is_gaussian = True

    def __init__(self, env, model_config, policy, policy_tag_to_agent_id_map,
                 create_separate_placeholders_for_each_policy=False,
                 obs_dim_corresponding_to_num_agents="first"):
        super().__init__(env, model_config, policy, policy_tag_to_agent_id_map,
                         create_separate_placeholders_for_each_policy,
                         obs_dim_corresponding_to_num_agents)
        assert self.is_deterministic, "fully_connected_gaussian needs a Box action space"
        self.log_std = nn.Parameter(torch.full(
            (self.flattened_action_size,), float(model_config.get("log_std_init", 0.0))))
        # the fused training forward is built for softmax heads
        self.use_fused_train_forward = False

    def forward(self, obs=None, action=None, action_mask=None):
        x = self.normalized_input(obs)
        for i in range(len(self.fc)):
            x = self.fc[str(i)](x)
        return [self.policy_head(x)], self.vf_head(x)[..., 0]


class ModelFactory:
    """type name -> model class (warp_drive/training/models/factory.py:37-59)."""

    _registry = {"fully_connected": FullyConnected,
                 "fully_connected_gaussian": FullyConnectedGaussian}

    @classmethod
    def add(cls, model_name, model_cls):
        cls._registry[model_name] = model_cls

    @classmethod
    def create(cls, model_name):
        if model_name == "fully_connected_q" and model_name not in cls._registry:
            # DQN's Q network, imported on first use
            from warp_drive_b200.training.models.fully_connected_q import FullyConnectedQ

            cls._registry[model_name] = FullyConnectedQ
        if model_name == "fully_connected_quantile_q" and model_name not in cls._registry:
            # QR-DQN's distributional Q network, imported on first use
            from warp_drive_b200.training.models.fully_connected_q import (
                FullyConnectedQuantileQ)

            cls._registry[model_name] = FullyConnectedQuantileQ
        if model_name == "fully_connected_iqn" and model_name not in cls._registry:
            # IQN's implicit quantile network, imported on first use
            from warp_drive_b200.training.models.fully_connected_q import FullyConnectedIQN

            cls._registry[model_name] = FullyConnectedIQN
        if model_name == "fully_connected_categorical_q" and model_name not in cls._registry:
            # C51's categorical Q network, imported on first use
            from warp_drive_b200.training.models.fully_connected_q import (
                FullyConnectedCategoricalQ)

            cls._registry[model_name] = FullyConnectedCategoricalQ
        if model_name == "fully_connected_branching_q" and model_name not in cls._registry:
            # branching DQN's Q network (one head per action dimension), imported on first use
            from warp_drive_b200.training.models.fully_connected_q import (
                FullyConnectedBranchingQ)

            cls._registry[model_name] = FullyConnectedBranchingQ
        if model_name == "fully_connected_gru" and model_name not in cls._registry:
            # the recurrent A2C / PPO policy, imported on first use
            from warp_drive_b200.training.models.fully_connected_gru import FullyConnectedGRU

            cls._registry[model_name] = FullyConnectedGRU
        if model_name == "fully_connected_gaussian_gru" and model_name not in cls._registry:
            # the recurrent Gaussian A2C / PPO policy for Box actions, imported on first use
            from warp_drive_b200.training.models.fully_connected_gru import (
                FullyConnectedGaussianGRU)

            cls._registry[model_name] = FullyConnectedGaussianGRU
        if model_name not in cls._registry and model_name in (
                "fully_connected_actor", "fully_connected_action_value_critic",
                "fully_connected_sac_actor", "fully_connected_quantile_critic"):
            # the DDPG pair (reference factory.py:10-16), SAC's actor and TQC's critic,
            # imported on first use
            from warp_drive_b200.training.models.fully_connected_actor_critic import (
                FullyConnectedActionValueCritic, FullyConnectedActor,
                FullyConnectedQuantileCritic, FullyConnectedSACActor)

            cls._registry["fully_connected_actor"] = FullyConnectedActor
            cls._registry["fully_connected_action_value_critic"] = (
                FullyConnectedActionValueCritic)
            cls._registry["fully_connected_sac_actor"] = FullyConnectedSACActor
            cls._registry["fully_connected_quantile_critic"] = FullyConnectedQuantileCritic
        if model_name not in cls._registry:
            raise ValueError(f"unknown model type '{model_name}'")
        return cls._registry[model_name]
