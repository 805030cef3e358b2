"""Actor and action-value critic for DDPG on continuous (Box) action spaces.

Forward contracts and parameter names of the reference's FullyConnectedActor /
FullyConnectedActionValueCritic (warp_drive/training/models/
fully_connected_actor_critic.py:13-144) so its checkpoints load unchanged:
  actor  : `fc.{i}.0`, `policy_head`            forward(obs)         -> [actions per head]
  critic : `fc.{i}.0` (input = obs ++ action), `vf_head`
                                                forward(obs, action) -> Q values [..]
The deterministic head is `output_w * tanh(linear) + output_b` (model config keys of
single_pendulum.yaml / single_continuous_mountain_car.yaml)."""
import torch
from torch import nn

from warp_drive_b200.training.models.fully_connected import FullyConnected


class FullyConnectedActor(FullyConnected):
    name = "torch_fully_connected_actor"

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        del self.vf_head                 # include_value_head=False in the reference

    def forward(self, obs=None, action=None):
        x = obs
        for i in range(len(self.fc)):
            x = self.fc[str(i)](x)
        return self._policy_outputs(x)

    def _policy_outputs(self, x):
        from torch.nn import functional as func

        from warp_drive_b200.training.models.fully_connected import apply_logit_mask

        if self.is_deterministic:
            out = torch.tanh(apply_logit_mask(self.policy_head(x), self.action_mask))
            out = self.action_scale * out + self.action_bias
            if self.output_dims[0] > 1:
                return [t.contiguous() for t in torch.split(out, 1, dim=-1)]
            return [out]
        masks = [None] * len(self.output_dims)
        if self.action_mask is not None:
            start = 0
            for k, dim in enumerate(self.output_dims):
                masks[k] = self.action_mask[..., start:start + dim]
                start += dim
        return [func.softmax(apply_logit_mask(head(x), masks[k]), dim=-1)
                for k, head in enumerate(self.policy_head)]


def squashed_log_prob(u, log_std, eps):
    """log pi of the tanh-squashed diagonal Gaussian at tanh(u), u = mu + exp(log_std) * eps,
    summed over the last dimension: the Gaussian density of u and the stable form
    2 (log 2 - u - softplus(-2 u)) of log(1 - tanh(u)^2).  The action scale does not enter."""
    import math

    from torch.nn import functional as func

    terms = (-0.5 * eps * eps - log_std - 0.5 * math.log(2 * math.pi)
             - 2.0 * (math.log(2.0) - u - func.softplus(-2.0 * u)))
    return terms.sum(dim=-1)


class FullyConnectedSACActor(FullyConnectedActor):
    """SAC's actor: the FullyConnectedActor trunk and one `policy_head = Linear(H, 2A)`, whose
    columns [0, A) are the mean mu and [A, 2A) the raw log-std, clamped to [log_std_min,
    log_std_max] (model config keys, default -20 and 2).  `forward(obs)` is the deterministic
    action [scale * tanh(mu) + bias] in the FullyConnectedActor contract (the evaluator plays
    it); `mean_and_log_std(obs)` is what the sampler and the update use."""

    name = "torch_fully_connected_sac_actor"
    is_squashed_gaussian = True

    def __init__(self, env, model_config, *args, **kwargs):
        super().__init__(env, model_config, *args, **kwargs)
        assert self.is_deterministic, "fully_connected_sac_actor needs a Box action space"
        self.log_std_min = float(model_config.get("log_std_min", -20.0))
        self.log_std_max = float(model_config.get("log_std_max", 2.0))
        assert self.log_std_min <= self.log_std_max
        A = self.output_dims[0]
        self.policy_head = nn.Linear(self.fc_dims[-1], 2 * A)

    def head_output(self, obs):
        """The head's raw output [..., 2A] (mu ++ unclamped log-std), what
        wdb_sample_squashed_gaussian reads."""
        x = obs
        for i in range(len(self.fc)):
            x = self.fc[str(i)](x)
        return self.policy_head(x)

    def mean_and_log_std(self, obs):
        z = self.head_output(obs)
        A = self.output_dims[0]
        return z[..., :A], z[..., A:].clamp(self.log_std_min, self.log_std_max)

    def squash(self, u):
        return self.action_scale * torch.tanh(u) + self.action_bias

    def sample(self, obs, eps):
        """(a = scale tanh(mu + sigma eps) + bias [..., A], log pi(a | obs) [...]) for standard
        normals eps [..., A], differentiable in the actor's parameters."""
        mu, log_std = self.mean_and_log_std(obs)
        u = mu + log_std.exp() * eps
        return self.squash(u), squashed_log_prob(u, log_std, eps)

    def forward(self, obs=None, action=None):
        mu, _ = self.mean_and_log_std(obs)
        out = self.squash(mu)
        if self.output_dims[0] > 1:
            return [t.contiguous() for t in torch.split(out, 1, dim=-1)]
        return [out]


class FullyConnectedActionValueCritic(FullyConnected):
    name = "torch_fully_connected_q"

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        del self.policy_head             # include_policy_head=False in the reference
        dims = [self.flattened_obs_size + self.flattened_action_size] + self.fc_dims
        self.fc = nn.ModuleDict({
            str(i): nn.Sequential(nn.Linear(dims[i], dims[i + 1]), nn.ReLU())
            for i in range(len(self.fc_dims))})

    def forward(self, obs=None, action=None):
        assert action is not None
        parts = [obs] + (list(action) if isinstance(action, (list, tuple)) else [action])
        x = torch.cat(parts, dim=-1)
        for i in range(len(self.fc)):
            x = self.fc[str(i)](x)
        return self.vf_head(x)[..., 0]


class FullyConnectedQuantileCritic(FullyConnectedActionValueCritic):
    """TQC's distributional critic: the FullyConnectedActionValueCritic trunk on obs ++ action
    and a raw `vf_head = Linear(H, N)`, N = model config key `num_quantiles` (default 25, an
    integer in [2, 64]).  `forward(obs, action)` is the N quantiles [..., N] at the midpoint
    fractions (2i + 1) / (2N)."""

    name = "torch_fully_connected_quantile_critic"

    def __init__(self, env, model_config, *args, **kwargs):
        n = model_config.get("num_quantiles", 25)
        if isinstance(n, bool) or not isinstance(n, int) or not 2 <= n <= 64:
            raise ValueError(f"num_quantiles must be an integer in [2, 64], got {n!r}")
        super().__init__(env, model_config, *args, **kwargs)
        self.num_quantiles = n
        self.vf_head = nn.Linear(self.fc_dims[-1], n)

    def forward(self, obs=None, action=None):
        assert action is not None
        parts = [obs] + (list(action) if isinstance(action, (list, tuple)) else [action])
        x = torch.cat(parts, dim=-1)
        for i in range(len(self.fc)):
            x = self.fc[str(i)](x)
        return self.vf_head(x)


class QuantileCritics(nn.Module):
    """TQC's M quantile critics as one module: what the critic optimizer steps (and clips by
    their joint norm) and the `{policy}_critic_{t}` checkpoint holds.  `forward(obs, action)` is
    [..., M, N]."""

    def __init__(self, critics):
        super().__init__()
        self.critics = nn.ModuleList(critics)

    def __len__(self):
        return len(self.critics)

    def __getitem__(self, m):
        return self.critics[m]

    def forward(self, obs=None, action=None):
        return torch.stack([c(obs=obs, action=action) for c in self.critics], dim=-2)


class ActorAsPolicy(nn.Module):
    """Adapter for the rollout engine, whose forward contract is `(probs, values)`.  A
    squashed-Gaussian actor hands the engine its raw head output [mu ++ log-std], which
    CUDASampler.sample_squashed_gaussian turns into actions."""

    def __init__(self, actor):
        super().__init__()
        self.actor = actor
        self.is_squashed_gaussian = bool(getattr(actor, "is_squashed_gaussian", False))

    def forward(self, obs=None):
        if self.is_squashed_gaussian:
            return [self.actor.head_output(obs)], None
        return self.actor(obs), None
