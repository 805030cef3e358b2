"""FullyConnectedQ: the Q network of DQN (training/trainer_dqn.py) for one Discrete(A) action.

The FullyConnected trunk (`fc_dims`: Linear + ReLU layers, module names `fc.{i}.0`) and one
raw `policy_head = Linear(fc_dims[-1], A)`: Q(obs, .) for every action, no softmax and no value
head.  `q_values(obs)` is what the update uses; `forward(obs)` keeps the rollout engine's
`(outputs per head, values)` contract as `([Q], None)`, and the engine recognises the network
by `is_q_network` and samples its actions epsilon-greedily (CUDASampler.sample_epsilon_greedy).
"""
from torch import nn
from torch.nn import functional as func

from warp_drive_b200.training.utils.data_loader import (
    action_head_sizes, dict_observation_keys, get_flattened_obs_size)
from warp_drive_b200.utils.spaces import Discrete


class FullyConnectedQ(nn.Module):
    name = "torch_fully_connected_q"
    is_q_network = True
    is_deterministic = False
    action_mask = None

    def __init__(self, env, model_config, policy, policy_tag_to_agent_id_map,
                 create_separate_placeholders_for_each_policy=False,
                 obs_dim_corresponding_to_num_agents="first"):
        super().__init__()
        self.fc_dims = list(model_config["fc_dims"])
        self.policy = policy
        sample_agent = policy_tag_to_agent_id_map[policy][0]
        self.observation_space = env.env.observation_space[sample_agent]
        action_space = env.env.action_space[sample_agent]
        if not isinstance(action_space, Discrete):
            raise ValueError("fully_connected_q takes a single Discrete action head, got "
                             f"{type(action_space).__name__}")
        heads, _ = action_head_sizes(action_space)
        _, masked = dict_observation_keys(self.observation_space)
        if masked:
            raise ValueError("fully_connected_q does not take observations with an action_mask")
        self.flattened_obs_size = get_flattened_obs_size(self.observation_space)
        self.output_dims = [int(heads[0])]
        dims = [self.flattened_obs_size] + self.fc_dims
        self.fc = nn.ModuleDict({
            str(i): nn.Sequential(nn.Linear(dims[i], dims[i + 1]), nn.ReLU())
            for i in range(len(self.fc_dims))})
        self.policy_head = nn.Linear(dims[-1], self.output_dims[0])

    def q_values(self, obs):
        """Q(obs, a) for every action: [..., A]."""
        x = obs
        for i in range(len(self.fc)):
            x = self.fc[str(i)](x)
        return self.policy_head(x)

    def forward(self, obs=None, action=None, action_mask=None):
        return [self.q_values(obs)], None


class FullyConnectedQuantileQ(FullyConnectedQ):
    """The distributional Q network of quantile-regression DQN (algorithms/dqn.py QuantileDQN,
    Dabney et al. 2018): FullyConnectedQ's trunk and one raw `policy_head = Linear(H, A * N)`,
    N = `num_quantiles` (an integer in [2, 256]); column a * N + i is quantile i of action a.
    `quantiles(obs)` is what the update uses; `q_values(obs)` -- and so `forward` and the
    rollout's epsilon-greedy actions -- is the mean over the quantiles, computed through the
    collapsed head (`collapsed_head()`: W and b averaged over each action's N rows)."""
    name = "torch_fully_connected_quantile_q"
    is_quantile_q = True

    def __init__(self, env, model_config, policy, policy_tag_to_agent_id_map,
                 create_separate_placeholders_for_each_policy=False,
                 obs_dim_corresponding_to_num_agents="first"):
        n = model_config.get("num_quantiles")
        if isinstance(n, bool) or not isinstance(n, int) or not 2 <= n <= 256:
            raise ValueError("fully_connected_quantile_q needs model.num_quantiles, an integer in "
                             f"[2, 256], got {n!r}")
        super().__init__(env, model_config, policy, policy_tag_to_agent_id_map,
                         create_separate_placeholders_for_each_policy,
                         obs_dim_corresponding_to_num_agents)
        self.num_quantiles = n
        self.policy_head = nn.Linear(self.policy_head.in_features, self.output_dims[0] * n)

    def trunk(self, obs):
        x = obs
        for i in range(len(self.fc)):
            x = self.fc[str(i)](x)
        return x

    def quantiles(self, obs):
        """The N quantiles of every action: [..., A, N]."""
        y = self.policy_head(self.trunk(obs))
        return y.reshape(*y.shape[:-1], self.output_dims[0], self.num_quantiles)

    def collapsed_head(self):
        """(W.view(A, N, H).mean(1), b.view(A, N).mean(1)): the head of the mean quantile."""
        A, n = self.output_dims[0], self.num_quantiles
        w, b = self.policy_head.weight, self.policy_head.bias
        return w.view(A, n, w.shape[1]).mean(1), b.view(A, n).mean(1)

    def q_values(self, obs):
        """The mean quantile of every action: [..., A]."""
        w, b = self.collapsed_head()
        return func.linear(self.trunk(obs), w, b)
