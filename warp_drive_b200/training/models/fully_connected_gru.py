"""FullyConnectedGRU: a recurrent policy for A2C / PPO.

The FullyConnected trunk (`fc_dims`, Linear + ReLU, modules `fc.{i}.0`; it may be empty), then an
`nn.GRUCell` of width `gru_dim` (model key, default `fc_dims[-1]`; module `gru`, parameters
`gru.weight_ih [3H, D]`, `gru.weight_hh [3H, H]`, `gru.bias_ih`, `gru.bias_hh`, gate order r, z,
n), then one softmax `policy_head.{k}` per discrete action head and the scalar `vf_head`, both
reading the GRU's new state h'.

The state a timestep starts from follows one rule (`reset_hidden`): h_in(0) is the recorded start
state of the batch, and h_in(t) = h_out(t - 1) * (1 - [done(t - 1) > 0]) with done the env's
`_done_flags_batch` row: an env that ended an episode at t - 1 starts the next one from zero.
The rollout (RolloutEngine) applies the same rule on the device with wdb_recurrent_reset_done.

* `step(obs [R, F], h [R, H]) -> ([probs per head] [R, A_k], h')`: one rollout step.
* `forward_sequence(obs [T, E, Np, F], h0 [E, Np, H], done_flags [T, E])
  -> ([probs per head] [T, E, Np, A_k], values [T, E, Np])`: the training forward, a loop over T
  under autograd (truncated backpropagation through time over the batch).

Discrete or MultiDiscrete actions; Box or Dict observations without an action mask.  Refused with
a ValueError: Box actions, an action mask, `normalize_observations` (and, in the trainer, any
algorithm but A2C / PPO).  `forward(obs)` refuses as well: a memoryless call would silently drop
the recurrence.

FullyConnectedGaussianGRU (`fully_connected_gaussian_gru`) is the same recurrent core for a 1-D
Box action space of A dimensions, as FullyConnectedGaussian is FullyConnected's: `policy_head` is
one Linear(H, A) whose raw output is the mean, and `log_std` a state-independent parameter [A]
(`log_std_init`, default 0).  Its `step` and `forward_sequence` return [mean] where the
categorical model returns its probabilities.
"""
import torch
from torch import nn
from torch.nn import functional as func

from warp_drive_b200.training.models.fully_connected import FullyConnected
from warp_drive_b200.training.utils.data_loader import (
    action_head_sizes, get_flattened_obs_size)
from warp_drive_b200.utils.constants import Constants
from warp_drive_b200.utils.spaces import Dict

_PROCESSED_OBSERVATIONS = Constants.PROCESSED_OBSERVATIONS
_ACTION_MASK = Constants.ACTION_MASK


class FullyConnectedGRU(FullyConnected):
    name = "torch_fully_connected_gru"
    model_type = "fully_connected_gru"
    is_recurrent = True
    normalize_observations = False
    # the fused training node and every feed-forward rollout kernel take memoryless models only
    use_fused_train_forward = False

    def __init__(self, env, model_config, policy, policy_tag_to_agent_id_map,
                 create_separate_placeholders_for_each_policy=False,
                 obs_dim_corresponding_to_num_agents="first"):
        nn.Module.__init__(self)
        self.env = env
        self.fc_dims = [int(d) for d in model_config.get("fc_dims", [])]
        self.policy = policy
        self.policy_tag_to_agent_id_map = policy_tag_to_agent_id_map
        self.create_separate_placeholders_for_each_policy = (
            create_separate_placeholders_for_each_policy)
        assert obs_dim_corresponding_to_num_agents in ("first", "last")
        self.obs_dim_corresponding_to_num_agents = obs_dim_corresponding_to_num_agents
        sample_agent = policy_tag_to_agent_id_map[policy][0]
        self.observation_space = env.env.observation_space[sample_agent]
        heads, self.is_deterministic = action_head_sizes(env.env.action_space[sample_agent])
        self._check_action_space(self.is_deterministic)
        kind = self.model_type
        if isinstance(self.observation_space, Dict) and _ACTION_MASK in self.observation_space:
            raise ValueError(f"{kind} does not take an action mask")
        if model_config.get("normalize_observations", False):
            raise ValueError(f"{kind} does not take normalize_observations")
        if not self.fc_dims and "gru_dim" not in model_config:
            raise ValueError(f"{kind} needs fc_dims or gru_dim")
        self.hidden_size = int(model_config.get("gru_dim", self.fc_dims[-1] if self.fc_dims
                                                else 0))
        if self.hidden_size < 1:
            raise ValueError(f"gru_dim must be at least 1, got {self.hidden_size}")
        self.flattened_obs_size = get_flattened_obs_size(self.observation_space)
        self.flattened_action_size = len(heads)
        self.output_dims = list(heads)
        dims = [self.flattened_obs_size] + self.fc_dims
        self.fc = nn.ModuleDict({
            str(i): nn.Sequential(nn.Linear(dims[i], dims[i + 1]), nn.ReLU())
            for i in range(len(self.fc_dims))})
        self.gru = nn.GRUCell(dims[-1], self.hidden_size)
        self._build_policy_head(heads)
        self.vf_head = nn.Linear(self.hidden_size, 1)
        self.action_mask = None
        name = f"{_PROCESSED_OBSERVATIONS}_batch_{policy}"
        self.batch_size = env.cuda_data_manager.get_shape(name=name)[0]

    @staticmethod
    def _check_action_space(is_box):
        if is_box:
            raise ValueError("fully_connected_gru takes Discrete or MultiDiscrete actions, "
                             "not a Box action space (fully_connected_gaussian_gru takes Box "
                             "actions)")

    def _build_policy_head(self, heads):
        self.policy_head = nn.ModuleList([nn.Linear(self.hidden_size, h) for h in heads])

    def forward(self, obs=None, action=None, action_mask=None):
        raise RuntimeError(f"{self.model_type} is recurrent: call step(obs, h) or "
                           "forward_sequence(obs, h0, done_flags)")

    def head_layers(self):
        """The policy head Linears, in output order."""
        return list(self.policy_head)

    # ---- the pieces
    def trunk(self, obs):
        x = obs
        for i in range(len(self.fc)):
            x = self.fc[str(i)](x)
        return x

    def heads(self, h):
        return [func.softmax(head(h), dim=-1) for head in self.policy_head]

    @staticmethod
    def reset_hidden(h, done_flags_row):
        """The state the next timestep starts from: h [E, Np, H] zeroed for every env whose
        done flag (a `_done_flags_batch` row [E]) is > 0."""
        keep = (done_flags_row <= 0).to(h.dtype)
        return h * keep[:, None, None]

    # ---- the two forwards
    def step(self, obs, h):
        """obs [R, F], h [R, H] -> ([probs per head] [R, A_k], h' [R, H])."""
        h_new = self.gru(self.trunk(obs), h)
        return self.heads(h_new), h_new

    def forward_sequence(self, obs, h0, done_flags):
        """obs [T, E, Np, F], h0 [E, Np, H] (no gradient flows into it), done_flags [T, E] ->
        ([probs per head] [T, E, Np, A_k], values [T, E, Np])."""
        T, E, Np = obs.shape[:3]
        x = self.trunk(obs.reshape(T, E * Np, -1))
        h = h0.detach().reshape(E * Np, self.hidden_size)
        outs = []
        for t in range(T):
            if t > 0:
                h = self.reset_hidden(h.view(E, Np, -1), done_flags[t - 1]).view(E * Np, -1)
            h = self.gru(x[t], h)
            outs.append(h)
        hs = torch.stack(outs).view(T, E, Np, self.hidden_size)
        return self.heads(hs), self.vf_head(hs)[..., 0]


class FullyConnectedGaussianGRU(FullyConnectedGRU):
    """The recurrent diagonal Gaussian policy: FullyConnectedGRU's trunk, cell, reset rule and
    value head; `policy_head` = one Linear(H, A) whose raw output is the mean (no tanh, no
    scaling) and `log_std` a state-independent parameter [A] (model key `log_std_init`, default
    0).  `step(obs, h) -> ([mean [R, A]], h')`, `forward_sequence -> ([mean [T, E, Np, A]],
    values)`.  A 1-D Box action space only; actions are drawn unclipped by
    CUDASampler.sample_gaussian from the mean and log_std, and the env bounds them."""

    name = "torch_fully_connected_gaussian_gru"
    model_type = "fully_connected_gaussian_gru"
    is_gaussian = True

    def __init__(self, env, model_config, policy, policy_tag_to_agent_id_map,
                 create_separate_placeholders_for_each_policy=False,
                 obs_dim_corresponding_to_num_agents="first"):
        super().__init__(env, model_config, policy, policy_tag_to_agent_id_map,
                         create_separate_placeholders_for_each_policy,
                         obs_dim_corresponding_to_num_agents)
        self.log_std = nn.Parameter(torch.full(
            (self.output_dims[0],), float(model_config.get("log_std_init", 0.0))))

    @staticmethod
    def _check_action_space(is_box):
        if not is_box:
            raise ValueError("fully_connected_gaussian_gru takes a 1-D Box action space, not "
                             "Discrete or MultiDiscrete actions (fully_connected_gru takes "
                             "those)")

    def _build_policy_head(self, heads):
        # (a Box space of A dimensions arrives as A heads of size 1: one mean head of A)
        self.output_dims = [len(heads)]
        self.policy_head = nn.Linear(self.hidden_size, len(heads))

    def head_layers(self):
        return [self.policy_head]

    def heads(self, h):
        return [self.policy_head(h)]


class NativeGruStep:
    """FullyConnectedGRU.step as ONE wdb_gru_policy_forward launch (csrc/wdb_recurrent.cu): the
    trunk, the GRU cell (h' written over h in place) and the heads' softmax, fp32, straight into
    the sampler's probability buffers; for FullyConnectedGaussianGRU the mean head kind, which
    writes the raw mean [R, A] into the sampler's mean buffer.  The value head is not evaluated
    (the rollout never reads values).  It reads the parameters where they are, so an optimizer
    step needs no re-pack."""

    @staticmethod
    def shape_args(model):
        """(F, n_layers, d0, d1, H, n_heads, a0, a1) of wdb_gru_forward_bytes, or None.  A
        Gaussian model's mean head is one head of A."""
        if not getattr(model, "is_recurrent", False) or len(model.fc) > 2:
            return None
        if len(model.output_dims) not in (1, 2):
            return None
        dims = [int(d) for d in model.fc_dims] + [0, 0]
        heads = [int(a) for a in model.output_dims] + [0]
        return (int(model.flattened_obs_size), len(model.fc), dims[0], dims[1],
                int(model.hidden_size), len(model.output_dims), heads[0], heads[1])

    @classmethod
    def supported(cls, model):
        from warp_drive_b200 import lib as _lib

        args = cls.shape_args(model)
        return args is not None and _lib.load().wdb_gru_forward_bytes(*args) > 0

    # Measured on an H100 80GB HBM3 at 700 W (scripts/bench_recurrent.py): 0.047 ms against the
    # torch step's 0.140 ms at gridworld's 0.16 GFLOP step, but 1.89 ms against 1.02 ms at
    # TagContinuous's 15 GFLOP step, where cuBLAS outruns this kernel's CUDA-core sums.  The
    # engine routes a policy here only while its step stays under this many FLOPs (the torch
    # step costs about its launch overhead, 0.14 ms, up to ~1 GFLOP).  The mean head kind
    # crosses over at the same place: 0.082 ms against 0.163 ms at 0.58 GFLOP (10 000 rows,
    # F = 3, [64, 64], GRU 64, A = 1), 0.147 ms against 0.134 ms at 1.21 GFLOP.
    MAX_ROUTED_FLOPS = 1e9

    @classmethod
    def step_flops(cls, model, rows):
        F, n_layers, d0, d1, H, _, a0, a1 = cls.shape_args(model)
        dims = [F, d0, d1][:n_layers + 1]
        mac = sum(a * b for a, b in zip(dims[:-1], dims[1:])) + 3 * H * (dims[-1] + H)
        return 2.0 * rows * (mac + H * (a0 + a1))

    @classmethod
    def routed(cls, model, rows):
        """Whether the rollout engine takes this kernel for `rows` rows of the policy: where it
        takes the shape and beats the torch step (MAX_ROUTED_FLOPS)."""
        return cls.supported(model) and cls.step_flops(model, rows) <= cls.MAX_ROUTED_FLOPS

    def __init__(self, model):
        assert self.supported(model)
        self.model = model

    def __call__(self, obs, hidden, probs):
        """obs [R, F] and hidden [R, H] (or [E, Np, H]) float32 contiguous; probs: one
        [R, A_k] (or [E, Np, A_k]) buffer per head."""
        import ctypes

        from warp_drive_b200 import lib as _lib

        m = self.model
        F, n_layers, d0, d1, H, n_heads, a0, a1 = self.shape_args(m)
        a = _lib.GruForward()
        a.n_rows = hidden.numel() // H
        a.in_dim, a.n_layers, a.hidden_size, a.n_heads = F, n_layers, H, n_heads
        a.dims[0], a.dims[1], a.heads[0], a.heads[1] = d0, d1, a0, a1
        a.head_kind = (_lib.GRU_HEAD_MEAN if getattr(m, "is_gaussian", False)
                       else _lib.GRU_HEAD_SOFTMAX)
        assert obs.numel() == a.n_rows * F and obs.dtype == torch.float32
        a.obs, a.hidden = _lib.ptr(obs), _lib.ptr(hidden)
        for i in range(n_layers):
            lin = m.fc[str(i)][0]
            a.fc_weight[i], a.fc_bias[i] = _lib.ptr(lin.weight), _lib.ptr(lin.bias)
        g = m.gru
        a.weight_ih, a.weight_hh = _lib.ptr(g.weight_ih), _lib.ptr(g.weight_hh)
        a.bias_ih, a.bias_hh = _lib.ptr(g.bias_ih), _lib.ptr(g.bias_hh)
        for k, head in enumerate(m.head_layers()):
            assert probs[k].numel() == a.n_rows * head.out_features
            a.head_weight[k], a.head_bias[k] = _lib.ptr(head.weight), _lib.ptr(head.bias)
            a.probs[k] = _lib.ptr(probs[k])
        _lib.check(_lib.load().wdb_gru_policy_forward(_lib.stream_ptr(), ctypes.byref(a)),
                   "gru_policy_forward")
