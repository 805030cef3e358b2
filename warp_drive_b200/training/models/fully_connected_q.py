"""FullyConnectedQ: the Q network of DQN (training/trainer_dqn.py) for one Discrete(A) action.

The FullyConnected trunk (`fc_dims`: Linear + ReLU layers, module names `fc.{i}.0`) and one
raw `policy_head = Linear(fc_dims[-1], A)`: Q(obs, .) for every action, no softmax and no value
head.  `q_values(obs)` is what the update uses; `forward(obs)` keeps the rollout engine's
`(outputs per head, values)` contract as `([Q], None)`, and the engine recognises the network
by `is_q_network` and samples its actions epsilon-greedily (CUDASampler.sample_epsilon_greedy).

Dueling (Wang et al. 2016): with the model key `dueling: true` the head is a DuelingHead (value
and advantage streams combined by the mean rule) with `stream_fc_dims` ([] or [S]) hidden
layers per stream, for fully_connected_q and fully_connected_categorical_q.  Its forward has the
plain head's column layout, so everything that reads the head's outputs works unchanged.

Noisy networks (Fortunato et al. 2018): with the model key `noisy: true` every Linear layer of the
head -- the plain head's output layer, or every stream layer of a DuelingHead -- is a NoisyLinear
with factorized Gaussian noise (`noisy_sigma0`, 0.5 by default); the trunk stays plain.  A layer
uses noise only while its `noise` is set (the update's sample, or per-row acting noise), and is
the mean network otherwise, so the evaluator plays the mean network.

Action branching (Tavakoli, Pardo & Kormushev 2018): FullyConnectedBranchingQ
(`fully_connected_branching_q`) takes a MultiDiscrete space (or one Discrete head) and puts one Q
head per action dimension on the shared trunk, as column blocks of one raw Linear.

Action masks: the model key `masked: true` over a Dict observation space with an `action_mask`
key of width A sets `masked` (without the key such a space is refused, as before).  The
mask is not a model input (`flattened_obs_size` excludes it) and the Q values stay raw: the
rollout's epsilon-greedy sampler acts over the valid actions
(CUDASampler.sample_epsilon_greedy's `action_mask`) and the losses bootstrap over the valid
actions of obs' (algorithms/dqn.py's `boot_mask`).
"""
import math

import torch
from torch import nn
from torch.nn import functional as func

from warp_drive_b200.training.utils.data_loader import (
    action_head_sizes, dict_observation_keys, get_flattened_obs_size)
from warp_drive_b200.utils.constants import Constants
from warp_drive_b200.utils.spaces import Discrete, MultiDiscrete

_ACTION_MASK = Constants.ACTION_MASK


def dueling_settings(model_config, model_type):
    """(dueling, stream_fc_dims) of a Q model config, validated; `model_type` names the model in
    the messages."""
    dueling = model_config.get("dueling", False)
    if not isinstance(dueling, bool):
        raise ValueError(f"{model_type}'s model.dueling is true or false, got {dueling!r}")
    if "stream_fc_dims" not in model_config:
        return dueling, []
    dims = model_config["stream_fc_dims"]
    if not dueling:
        raise ValueError(f"{model_type}'s model.stream_fc_dims needs model.dueling: true, got "
                         f"stream_fc_dims {dims!r} without it")
    if not isinstance(dims, list) or len(dims) > 1 or not all(
            isinstance(d, int) and not isinstance(d, bool) and d > 0 for d in dims):
        raise ValueError(f"{model_type}'s model.stream_fc_dims is a list of at most one positive "
                         f"integer, got {dims!r}")
    return dueling, list(dims)


def noisy_settings(model_config, model_type):
    """(noisy, sigma0) of a Q model config, validated; `model_type` names the model in the
    messages."""
    noisy = model_config.get("noisy", False)
    if not isinstance(noisy, bool):
        raise ValueError(f"{model_type}'s model.noisy is true or false, got {noisy!r}")
    if "noisy_sigma0" not in model_config:
        return noisy, 0.5
    s = model_config["noisy_sigma0"]
    if not noisy:
        raise ValueError(f"{model_type}'s model.noisy_sigma0 needs model.noisy: true, got "
                         f"noisy_sigma0 {s!r} without it")
    if isinstance(s, bool) or not isinstance(s, (int, float)) or not math.isfinite(s) or s <= 0:
        raise ValueError(f"{model_type}'s model.noisy_sigma0 is a finite number > 0, got {s!r}")
    return noisy, float(s)


def masked_settings(model_config, observation_space, n_actions):
    """model.masked (bool, False) of a Q model config, validated against the observation space:
    an `action_mask` key is refused without `masked: true`, `masked: true` is refused without
    one, and the mask must have one entry per action."""
    masked = model_config.get("masked", False)
    if not isinstance(masked, bool):
        raise ValueError(f"a Q model's model.masked is true or false, got {masked!r}")
    _, has_mask = dict_observation_keys(observation_space)
    if has_mask and not masked:
        raise ValueError("fully_connected_q does not take observations with an action_mask "
                         "unless model.masked is true")
    if masked and not has_mask:
        raise ValueError("model.masked: true needs a Dict observation space with an "
                         f"{_ACTION_MASK!r} key")
    if masked:
        width = get_flattened_obs_size(observation_space[_ACTION_MASK])
        if width != n_actions:
            raise ValueError(f"a masked Q model's action_mask must have one entry per action "
                             f"({n_actions}), got width {width}")
    return masked


class NoisyLinear(nn.Module):
    """Linear(in, out) with factorized Gaussian noise (Fortunato et al. 2018):
        W = mu_W + sigma_W * (f(eps_out) f(eps_in)^T),  b = mu_b + sigma_b * f(eps_out),
    f(x) = sgn(x) sqrt(|x|).  mu ~ U(+-1/sqrt(in)), sigma = sigma0 / sqrt(in).  The f(eps)
    vectors of the update's sample are the non-persistent buffers `noise_in` [in] and
    `noise_out` [out] (written by wdb_noisy_materialize or wdb_noisy_draw; checkpoints hold the
    parameters only).  `noise` selects what forward uses: None (the mean network, mu only), the
    buffers' sample (W, b as materialized()), or per-row acting noise ([..., in], [..., out]
    matching the input's rows) in the factored form
        y = mu_W x + mu_b + f(eps_out) * (sigma_W (f(eps_in) * x) + sigma_b)."""
    is_noisy = True

    def __init__(self, in_features, out_features, sigma0=0.5):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        bound = 1.0 / math.sqrt(in_features)
        self.weight_mu = nn.Parameter(torch.empty(out_features, in_features).uniform_(-bound, bound))
        self.weight_sigma = nn.Parameter(torch.full((out_features, in_features), sigma0 * bound))
        self.bias_mu = nn.Parameter(torch.empty(out_features).uniform_(-bound, bound))
        self.bias_sigma = nn.Parameter(torch.full((out_features,), sigma0 * bound))
        self.register_buffer("noise_in", torch.zeros(in_features), persistent=False)
        self.register_buffer("noise_out", torch.zeros(out_features), persistent=False)
        self.noise = None

    def materialized(self, noise_in=None, noise_out=None):
        """(W, b) under the noise vectors (default: the buffers): the reference statement of
        wdb_noisy_materialize, differentiable in the parameters."""
        fi = self.noise_in if noise_in is None else noise_in
        fo = self.noise_out if noise_out is None else noise_out
        w = self.weight_mu + self.weight_sigma * (fo[:, None] * fi[None, :])
        b = self.bias_mu + self.bias_sigma * fo
        return w, b

    def forward(self, x):
        if self.noise is None:
            return func.linear(x, self.weight_mu, self.bias_mu)
        fi, fo = self.noise
        if fi.dim() == 1:
            return func.linear(x, *self.materialized(fi, fo))
        rows = x.shape[:-1]
        fi, fo = fi.reshape(*rows, -1), fo.reshape(*rows, -1)
        return (func.linear(x, self.weight_mu, self.bias_mu)
                + fo * func.linear(fi * x, self.weight_sigma, self.bias_sigma))


def linear_layer(in_features, out_features, sigma0=None):
    """nn.Linear, or a NoisyLinear when sigma0 is given."""
    if sigma0 is None:
        return nn.Linear(in_features, out_features)
    return NoisyLinear(in_features, out_features, sigma0)


def layer_params(layer):
    """(weight, bias) of a Linear, or a NoisyLinear's materialized() under its noise buffers."""
    if getattr(layer, "is_noisy", False):
        return layer.materialized()
    return layer.weight, layer.bias


class DuelingHead(nn.Module):
    """The dueling head (Wang et al. 2016) over a trunk output h of width H, for A actions of N
    outputs each (N = 1: Q values; N atoms: C51's logits).  Each stream has one hidden Linear(H,
    S) + ReLU when `stream_dim` S > 0, and reads h directly when S = 0:
        V = value(h) [..., N],  Adv = advantage(h) [..., A * N],
        out[a * N + j] = V_j + Adv[a * N + j] - (1/A) sum_c Adv[c * N + j]
    (the mean form of the paper's eq. 9), in the plain head's column layout [..., A * N].
    Parameters: `value.*` and `advantage.*` (Sequential(Linear, ReLU, Linear) or one Linear)."""
    is_dueling = True

    def __init__(self, in_features, n_actions, n_outputs, stream_dim, sigma0=None):
        super().__init__()
        self.in_features, self.n_actions, self.n_outputs = in_features, n_actions, n_outputs
        self.stream_dim = stream_dim
        self.out_features = n_actions * n_outputs

        def stream(width):       # sigma0: every stream layer is a NoisyLinear
            if stream_dim == 0:
                return linear_layer(in_features, width, sigma0)
            return nn.Sequential(linear_layer(in_features, stream_dim, sigma0), nn.ReLU(),
                                 linear_layer(stream_dim, width, sigma0))
        self.value = stream(n_outputs)
        self.advantage = stream(n_actions * n_outputs)

    def streams(self):
        """[(hidden, output)] Linear layers of the value and the advantage stream (hidden: None
        when S = 0)."""
        if self.stream_dim == 0:
            return [(None, self.value), (None, self.advantage)]
        return [(self.value[0], self.value[2]), (self.advantage[0], self.advantage[2])]

    def forward(self, h):
        A, N = self.n_actions, self.n_outputs
        v = self.value(h)
        adv = self.advantage(h)
        adv = adv.reshape(*adv.shape[:-1], A, N)
        out = v[..., None, :] + (adv - adv.mean(dim=-2, keepdim=True))
        return out.reshape(*out.shape[:-2], A * N)

    def folded(self):
        """[(weight, bias)] of the plain layers this head equals: the stacked stream hidden
        layer ([2S, H], S > 0) and the output layer [A * N, 2S or H] -- the reference statement of
        the fold (wdb_dueling_fold).  Differentiable in the stream parameters.  Noisy streams fold
        their materialized() layers."""
        A, N = self.n_actions, self.n_outputs
        (vh, vo), (ah, ao) = [tuple(None if x is None else layer_params(x) for x in pair)
                              for pair in self.streams()]

        def centred(x):                    # rows a * N + j minus the mean over a
            y = x.reshape(A, N, *x.shape[1:])
            return (y - y.mean(dim=0, keepdim=True)).reshape(x.shape)
        if self.stream_dim == 0:
            w = vo[0].repeat(A, 1) + centred(ao[0])
            b = vo[1].repeat(A) + centred(ao[1])
            return [(w, b)]
        hidden = (torch.cat([vh[0], ah[0]]), torch.cat([vh[1], ah[1]]))
        w = torch.cat([vo[0].repeat(A, 1), centred(ao[0])], dim=1)
        b = vo[1].repeat(A) + centred(ao[1])
        return [hidden, (w, b)]


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
        # `masked: true` with an `action_mask` key: the Q values stay raw, the sampler and the
        # losses apply the mask
        self.masked = masked_settings(model_config, self.observation_space, int(heads[0]))
        self.flattened_obs_size = get_flattened_obs_size(self.observation_space)
        self.output_dims = [int(heads[0])]
        dims = [self.flattened_obs_size] + self.fc_dims
        model_type = model_config.get("type", "fully_connected_q")
        self.dueling, self.stream_fc_dims = dueling_settings(model_config, model_type)
        self.noisy, self.noisy_sigma0 = noisy_settings(model_config, model_type)
        self.fc = nn.ModuleDict({
            str(i): nn.Sequential(nn.Linear(dims[i], dims[i + 1]), nn.ReLU())
            for i in range(len(self.fc_dims))})
        self.policy_head = self._head(dims[-1], 1)

    def _head(self, in_features, n_outputs):
        """The head of A * n_outputs raw outputs: one Linear, or a DuelingHead (noisy: of
        NoisyLinear layers)."""
        A = self.output_dims[0]
        sigma0 = self.noisy_sigma0 if self.noisy else None
        if self.dueling:
            return DuelingHead(in_features, A, n_outputs, sum(self.stream_fc_dims), sigma0)
        return linear_layer(in_features, A * n_outputs, sigma0)

    def noisy_layers(self):
        """The head's NoisyLinear layers in module order (the `layer` of their noise counter);
        [] for a plain network."""
        return [m for m in self.policy_head.modules() if getattr(m, "is_noisy", False)]

    def q_values(self, obs):
        """Q(obs, a) for every action: [..., A]."""
        x = obs
        for i in range(len(self.fc)):
            x = self.fc[str(i)](x)
        return self.policy_head(x)

    def forward(self, obs=None, action=None, action_mask=None):
        return [self.q_values(obs)], None


def _refuse_dueling(model_config, model_type):
    """QR-DQN's collapsed head and IQN's post-merge head would each need a fold of their own, and
    a noise map of their own."""
    for key in ("dueling", "stream_fc_dims"):
        if key in model_config and model_config[key] not in (False, None):
            raise ValueError(f"{model_type} does not take model.{key} (dueling heads are "
                             f"fully_connected_q's and fully_connected_categorical_q's), got "
                             f"{model_config[key]!r}")
    for key in ("noisy", "noisy_sigma0"):
        if key in model_config and model_config[key] not in (False, None):
            raise ValueError(f"{model_type} does not take model.{key} (noisy heads are "
                             f"fully_connected_q's and fully_connected_categorical_q's), got "
                             f"{model_config[key]!r}")


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
        _refuse_dueling(model_config, "fully_connected_quantile_q")
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


class FullyConnectedIQN(FullyConnectedQ):
    """The implicit quantile network of IQN (algorithms/dqn.py ImplicitQuantileDQN; Dabney,
    Ostrovski, Silver & Munos 2018): the return distribution as a function of the level tau.

    Trunk psi(x): FullyConnectedQ's `fc_dims` layers (at least one), width H.  Embedding
    phi(tau) = ReLU(`tau_embedding`(cos(pi i tau) for i = 0 .. n_cos - 1)), `tau_embedding` =
    Linear(n_cos, H) (i = 0 is the constant 1, as in the paper).  Value at level tau:
    Z_tau(x, .) = `policy_head`(psi(x) * phi(tau)), `policy_head` one raw Linear(H, A).  The paper
    puts one more hidden layer after the merge; here the head is one raw Linear, as QR-DQN's, so
    that acting collapses exactly into one Linear (below).

    Model keys (Dopamine's names; Dopamine calls n_cos `quantile_embedding_dim`):
    `num_cosines` n_cos (64, in [1, 64]), `num_tau_samples` N (32, in [1, 64]) and
    `num_tau_prime_samples` N' (32, in [1, 64]), the online and target levels per loss row, and
    `num_quantile_samples` K (32, in [1, 256]), the levels averaged for acting and for the
    bootstrap action.

    Acting averages Z over the fixed midpoints tau~_k = (2k + 1) / (2K) rather than over K fresh
    samples per step as the paper does -- a deliberate divergence that keeps it deterministic:
    Q(x, a) = mean_k Z_tau~k(x, a) = `policy_head`(psi(x) * c-bar), c-bar = mean_k phi(tau~_k),
    so `collapsed_head()` = (W diag(c-bar), b) is exact.  `q_values`, and through it `forward`,
    the per-step epsilon-greedy path, the one-launch rollout and the evaluator, go through it.
    `quantiles_at(x, taus)` is what the update uses."""
    name = "torch_fully_connected_iqn"
    is_implicit_quantile_q = True

    # (key, default, largest value); each is an integer of at least 1
    KEYS = (("num_cosines", 64, 64), ("num_tau_samples", 32, 64),
            ("num_tau_prime_samples", 32, 64), ("num_quantile_samples", 32, 256))

    def __init__(self, env, model_config, policy, policy_tag_to_agent_id_map,
                 create_separate_placeholders_for_each_policy=False,
                 obs_dim_corresponding_to_num_agents="first"):
        _refuse_dueling(model_config, "fully_connected_iqn")
        dims = model_config.get("fc_dims")
        if not dims:
            raise ValueError("fully_connected_iqn needs model.fc_dims with at least one hidden "
                             f"layer (the trunk the tau embedding multiplies), got {dims!r}")
        counts = {}
        for key, default, top in self.KEYS:
            v = model_config.get(key, default)
            if isinstance(v, bool) or not isinstance(v, int) or not 1 <= v <= top:
                raise ValueError(f"fully_connected_iqn's model.{key} is an integer in [1, {top}], "
                                 f"got {v!r}")
            counts[key] = v
        super().__init__(env, model_config, policy, policy_tag_to_agent_id_map,
                         create_separate_placeholders_for_each_policy,
                         obs_dim_corresponding_to_num_agents)
        for key, v in counts.items():
            setattr(self, key, v)
        self.tau_embedding = nn.Linear(self.num_cosines, self.policy_head.in_features)

    def trunk(self, obs):
        """psi(obs): [..., H]."""
        x = obs
        for i in range(len(self.fc)):
            x = self.fc[str(i)](x)
        return x

    def cos_features(self, taus):
        """cos(pi i tau) for i = 0 .. n_cos - 1: [..., n_cos].  pi i is rounded once to the
        levels' dtype, then multiplied by tau: the float32 operations of the native pass."""
        freq = math.pi * torch.arange(self.num_cosines, dtype=torch.float64, device=taus.device)
        return torch.cos(taus[..., None] * freq.to(taus.dtype))

    def embedding(self, taus):
        """phi(tau): [..., H]."""
        return func.relu(self.tau_embedding(self.cos_features(taus)))

    def quantiles_at(self, obs, taus):
        """Z at the given levels: obs [B, F], taus [B, T] (each row its own levels) or [T]
        (shared) -> [B, T, A]."""
        return self.policy_head(self.trunk(obs)[..., None, :] * self.embedding(taus))

    def acting_levels(self):
        """The K midpoints tau~_k = (2k + 1) / (2K) that acting and a* average over."""
        w = self.policy_head.weight
        k = self.num_quantile_samples
        return (2 * torch.arange(k, dtype=w.dtype, device=w.device) + 1) / (2 * k)

    def collapsed_head(self):
        """(W diag(c-bar), b), c-bar = mean_k phi(tau~_k): the head of the mean over the K
        midpoints."""
        cbar = self.embedding(self.acting_levels()).mean(0)
        return self.policy_head.weight * cbar, self.policy_head.bias

    def q_values(self, obs):
        """The mean of Z over the K midpoints, for every action: [..., A]."""
        w, b = self.collapsed_head()
        return func.linear(self.trunk(obs), w, b)


class FullyConnectedCategoricalQ(FullyConnectedQ):
    """The categorical Q network of C51 (algorithms/dqn.py CategoricalDQN; Bellemare, Dabney &
    Munos 2017): a softmax over N fixed atoms of the return per action.

    FullyConnectedQ's trunk and one raw `policy_head = Linear(H, A * N)`; column a * N + j is the
    logit of atom j of action a (QR-DQN's layout).  Model keys: `num_atoms` N (51, an integer in
    [2, 64]) and the required finite `v_min` < `v_max`.  The support z_j = v_min + j dz,
    dz = (v_max - v_min) / (N - 1), is computed in float64 and rounded once to float32; it is a
    non-persistent buffer (checkpoints hold the parameters only) and `delta_z` is dz rounded the
    same way, so the torch path and both native paths read the same values.

    `logits(obs)` [..., A, N] and `probabilities(obs)` (their softmax over the atoms) are what
    the update uses; `q_values(obs)` = sum_j z_j p_j [..., A] -- and so `forward`, the per-step
    epsilon-greedy path and the evaluator -- is the expectation.  The expectation is not linear
    in the head, so there is no collapsed_head()."""
    name = "torch_fully_connected_categorical_q"
    is_categorical_q = True

    def __init__(self, env, model_config, policy, policy_tag_to_agent_id_map,
                 create_separate_placeholders_for_each_policy=False,
                 obs_dim_corresponding_to_num_agents="first"):
        n = model_config.get("num_atoms", 51)
        if isinstance(n, bool) or not isinstance(n, int) or not 2 <= n <= 64:
            raise ValueError("fully_connected_categorical_q's model.num_atoms is an integer in "
                             f"[2, 64], got {n!r}")
        bounds = {}
        for key in ("v_min", "v_max"):
            v = model_config.get(key)
            if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v):
                raise ValueError(f"fully_connected_categorical_q needs model.{key}, a finite "
                                 f"number, got {v!r}")
            bounds[key] = float(v)
        if not bounds["v_min"] < bounds["v_max"]:
            raise ValueError("fully_connected_categorical_q needs model.v_min < model.v_max, got "
                             f"v_min {bounds['v_min']!r} and v_max {bounds['v_max']!r}")
        super().__init__(env, model_config, policy, policy_tag_to_agent_id_map,
                         create_separate_placeholders_for_each_policy,
                         obs_dim_corresponding_to_num_agents)
        self.num_atoms = n
        self.v_min, self.v_max = bounds["v_min"], bounds["v_max"]
        dz = (self.v_max - self.v_min) / (n - 1)
        support = self.v_min + dz * torch.arange(n, dtype=torch.float64)
        self.delta_z = float(torch.tensor(dz, dtype=torch.float64).float())
        self.register_buffer("support", support.float(), persistent=False)
        self.policy_head = self._head(self.policy_head.in_features, n)

    def trunk(self, obs):
        x = obs
        for i in range(len(self.fc)):
            x = self.fc[str(i)](x)
        return x

    def logits(self, obs):
        """The atom logits of every action: [..., A, N]."""
        y = self.policy_head(self.trunk(obs))
        return y.reshape(*y.shape[:-1], self.output_dims[0], self.num_atoms)

    def probabilities(self, obs):
        """The softmax over the atoms of every action: [..., A, N]."""
        return torch.softmax(self.logits(obs), dim=-1)

    def q_values(self, obs):
        """The expectation sum_j z_j p_j of every action: [..., A]."""
        p = self.probabilities(obs)
        return (p * self.support.to(p.dtype)).sum(dim=-1)


# the model keys of the other Q networks, which branching does not combine with
_BRANCHING_REFUSED = ("dueling", "stream_fc_dims", "noisy", "noisy_sigma0", "masked",
                      "num_quantiles", "num_cosines", "num_tau_samples", "num_tau_prime_samples",
                      "num_quantile_samples", "num_atoms", "v_min", "v_max")


class FullyConnectedBranchingQ(nn.Module):
    """The Q network of branching DQN (algorithms/dqn.py BranchingDQN; Tavakoli, Pardo &
    Kormushev 2018, "Action Branching Architectures for Deep Reinforcement Learning") for a
    MultiDiscrete action space, or one Discrete head (D = 1).

    FullyConnectedQ's trunk (`fc.{i}.0`) and ONE raw `policy_head = Linear(H, A)`,
    A = sum_d A_d over the heads' sizes `branch_sizes`: head d's Q values are columns
    o_d .. o_d + A_d - 1, o_d = A_0 + ... + A_{d-1}, so the outputs grow with the sum of the head
    sizes, not their product.  The module names and parameter creation order are
    FullyConnectedQ's, so at D = 1 the same seed gives the same weights and a checkpoint loads
    into either type.  `q_values` returns [..., A] and `forward` `([Q], None)`; the rollout
    samples each head epsilon-greedily on its own (CUDASampler.sample_epsilon_greedy with
    `branch_sizes`).

    Refused: Box actions, an `action_mask`, and the keys of the other Q networks (dueling, noisy,
    masked, quantile, IQN and C51 heads)."""
    name = "torch_fully_connected_branching_q"
    is_q_network = True
    is_branching_q = True
    is_deterministic = False
    action_mask = None
    masked = dueling = noisy = False

    def __init__(self, env, model_config, policy, policy_tag_to_agent_id_map,
                 create_separate_placeholders_for_each_policy=False,
                 obs_dim_corresponding_to_num_agents="first"):
        super().__init__()
        for key in _BRANCHING_REFUSED:
            if key in model_config and model_config[key] not in (False, None):
                raise ValueError(f"fully_connected_branching_q does not take model.{key}, got "
                                 f"{model_config[key]!r}")
        self.fc_dims = list(model_config["fc_dims"])
        self.policy = policy
        sample_agent = policy_tag_to_agent_id_map[policy][0]
        self.observation_space = env.env.observation_space[sample_agent]
        action_space = env.env.action_space[sample_agent]
        if not isinstance(action_space, (Discrete, MultiDiscrete)):
            raise ValueError("fully_connected_branching_q takes a Discrete or MultiDiscrete "
                             f"action space, got {type(action_space).__name__}")
        if dict_observation_keys(self.observation_space)[1]:
            raise ValueError("fully_connected_branching_q does not take observations with an "
                             "action_mask")
        heads, _ = action_head_sizes(action_space)
        self.branch_sizes = [int(a) for a in heads]
        self.output_dims = list(self.branch_sizes)
        self.flattened_obs_size = get_flattened_obs_size(self.observation_space)
        dims = [self.flattened_obs_size] + self.fc_dims
        self.fc = nn.ModuleDict({
            str(i): nn.Sequential(nn.Linear(dims[i], dims[i + 1]), nn.ReLU())
            for i in range(len(self.fc_dims))})
        self.policy_head = nn.Linear(dims[-1], sum(self.branch_sizes))

    def noisy_layers(self):
        return []

    def branches(self, q):
        """Q [..., A] split into the heads' Q values [[..., A_d] per head]."""
        return list(torch.split(q, self.branch_sizes, dim=-1))

    def q_values(self, obs):
        """Every head's Q values, side by side: [..., A]."""
        x = obs
        for i in range(len(self.fc)):
            x = self.fc[str(i)](x)
        return self.policy_head(x)

    def forward(self, obs=None, action=None, action_mask=None):
        return [self.q_values(obs)], None
