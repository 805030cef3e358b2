"""Fused DDPG update: `wdb_ddpg_update` (csrc/wdb_ddpg_update.cu) computes every actor and
critic gradient of one TrainerDDPG update from the replay ring in place -- five forwards, the
n-step returns, both losses and both backward passes -- and writes them straight into the
`.grad` views of the gradient arena; the counterpart of fused_loss.py for A2C / PPO.  The
torch autograd update (trainer_ddpg.py) stays for the shapes this does not take."""
import ctypes

import torch

from warp_drive_b200 import lib as _lib
from warp_drive_b200.utils.spaces import Box


def _layers(model):
    """[(weight, bias)] of the hidden Linear layers, then the head (actor: policy_head,
    critic: vf_head)."""
    head = model.policy_head if hasattr(model, "policy_head") else model.vf_head
    if getattr(head, "is_dueling", False):
        raise TypeError("a dueling head has no one output layer: the native passes run its "
                        "folded layers (fused_dqn.FusedDuelingUpdate)")
    if getattr(head, "is_noisy", False):
        raise TypeError("a noisy head has no one weight: the native passes run its "
                        "materialized layers (fused_dqn.FusedNoisyUpdate)")
    return [(model.fc[str(i)][0].weight, model.fc[str(i)][0].bias)
            for i in range(len(model.fc))] + [(head.weight, head.bias)]


def _set_shape(net, model):
    widths = [int(w) for w in model.fc_dims]
    net.n_hidden = len(widths)
    for i, w in enumerate(widths):
        net.widths[i] = w


def _set_pointers(net, model, grads):
    for i, (w, b) in enumerate(_layers(model)):
        net.w[i], net.b[i] = _lib.ptr(w.data), _lib.ptr(b.data)
        if grads:
            net.gw[i], net.gb[i] = _lib.ptr(w.grad), _lib.ptr(b.grad)


def _shape_struct(actor, critic, n_envs, n_agents, capacity, n_step):
    u = _lib.DdpgUpdate()
    u.n_envs, u.n_agents = int(n_envs), int(n_agents)
    u.obs_dim = int(actor.flattened_obs_size)
    u.action_dim = int(actor.output_dims[0])
    u.capacity, u.cursor, u.n_step = int(capacity), 0, int(n_step)
    for net, model in ((u.actor, actor), (u.critic, critic), (u.target_actor, actor),
                       (u.target_critic, critic)):
        _set_shape(net, model)
    return u


def fused_ddpg_supported(algo, actor, critic, n_envs, n_agents, capacity, n_step,
                         replay_rows=None):
    """True if `wdb_ddpg_update` takes this policy: a FullyConnectedActor (tanh head, Box
    observation, no action mask) and a FullyConnectedActionValueCritic of 0..3 hidden layers of
    width <= 64, obs + action width <= 64, and no return normalisation.  replay_rows: asks
    `wdb_ddpg_update_sampled` with that many sampled windows per update instead."""
    if not fused_models_supported(algo, actor, critic):
        return False
    u = _shape_struct(actor, critic, n_envs, n_agents, capacity, n_step)
    if replay_rows is not None:
        return bool(_lib.load().wdb_ddpg_update_sampled_supported(ctypes.byref(u), replay_rows))
    return bool(_lib.load().wdb_ddpg_update_supported(ctypes.byref(u)))


def replay_windows(windows):
    """struct wdb_replay_windows of a device int32 tensor [B, 2] (physical start slot, agent
    row), as wdb_replay_sample_windows writes it."""
    assert windows.dtype == torch.int32 and windows.dim() == 2 and windows.shape[1] == 2
    w = _lib.ReplayWindows()
    w.windows, w.n_windows = _lib.ptr(windows), int(windows.shape[0])
    return w


def fused_models_supported(algo, actor, critic, actor_type=None):
    """The model and algorithm checks of the fused actor-critic updates (DDPG, TD3, SAC with
    actor_type FullyConnectedSACActor); the kernels' own support calls check the shapes."""
    from warp_drive_b200.training.models.fully_connected_actor_critic import (
        FullyConnectedActionValueCritic, FullyConnectedActor)

    if algo.normalize_return:
        return False
    if type(actor) is not (actor_type or FullyConnectedActor) or type(critic) is not (
            FullyConnectedActionValueCritic):
        return False
    if not actor.is_deterministic or actor.action_mask is not None:
        return False
    if not isinstance(actor.observation_space, Box) or not isinstance(
            critic.observation_space, Box):
        return False
    if len(actor.fc_dims) > 3 or len(critic.fc_dims) > 3:
        return False
    return critic.flattened_obs_size == actor.flattened_obs_size


class FusedDDPGUpdate:
    """One policy's `wdb_ddpg_update` launch: the argument struct, its workspace and the loss
    sums (device double[2]: sum (Q - R)^2, sum J)."""

    def __init__(self, actor, critic, target_actor, target_critic, n_envs, n_agents,
                 capacity, n_step, gamma, replay_rows=None):
        self.models = (actor, critic, target_actor, target_critic)
        u = self.u = _shape_struct(actor, critic, n_envs, n_agents, capacity, n_step)
        u.gamma = float(gamma)
        u.action_scale, u.action_bias = float(actor.action_scale), float(actor.action_bias)
        self.lib = _lib.load()
        if replay_rows is None:
            nbytes = int(self.lib.wdb_ddpg_update_workspace_bytes(ctypes.byref(u)))
        else:
            nbytes = int(self.lib.wdb_ddpg_update_sampled_workspace_bytes(
                ctypes.byref(u), replay_rows))
        assert nbytes > 0, "shapes not supported by wdb_ddpg_update"
        dev = next(actor.parameters()).device
        self.workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        self.sums = torch.zeros(2, dtype=torch.float64, device=dev)
        self.valid = int(capacity) - int(n_step) + 1
        # loss rows per update: every window of the ring, or replay_rows sampled windows
        self.rows = self.valid * int(n_envs) * int(n_agents) if replay_rows is None else int(
            replay_rows)

    def launch(self, obs, actions, rewards, done, cursor, outputs=None, windows=None):
        """Gradients of the update into the actor's and the critic's `.grad`.  obs [C, E, Np,
        F], actions [C, E, Np, A], rewards [C, E, Np], done [C, E] are the ring in physical slot
        order, `cursor` its oldest slot.  outputs: optional (values, j_values, returns) tensors
        [valid, E, Np] for the metrics.  windows: int32 [rows, 2] sampled windows -- the update
        runs over them (wdb_ddpg_update_sampled; `cursor` is not read, outputs are [rows])."""
        u = self.u
        actor, critic, target_actor, target_critic = self.models
        # parameters may have been re-allocated (load_state_dict keeps storage; .to() does not)
        _set_pointers(u.actor, actor, True)
        _set_pointers(u.critic, critic, True)
        _set_pointers(u.target_actor, target_actor, False)
        _set_pointers(u.target_critic, target_critic, False)
        u.cursor = int(cursor)
        u.obs, u.actions = _lib.ptr(obs), _lib.ptr(actions)
        u.rewards, u.done = _lib.ptr(rewards), _lib.ptr(done)
        values, j_values, returns = outputs if outputs is not None else (None, None, None)
        u.values, u.j_values, u.returns = _lib.ptr(values), _lib.ptr(j_values), _lib.ptr(returns)
        u.sums = _lib.ptr(self.sums)
        u.workspace = _lib.ptr(self.workspace)
        if windows is not None:
            assert windows.shape[0] == self.rows
            _lib.check(self.lib.wdb_ddpg_update_sampled(
                _lib.stream_ptr(), ctypes.byref(u), ctypes.byref(replay_windows(windows))),
                "ddpg_update_sampled")
        else:
            _lib.check(self.lib.wdb_ddpg_update(_lib.stream_ptr(), ctypes.byref(u)),
                       "ddpg_update")
        return self.sums
