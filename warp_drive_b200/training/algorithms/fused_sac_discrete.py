"""Fused discrete SAC update: `wdb_sac_discrete_critic_update_sampled` and
`wdb_sac_discrete_actor_update_sampled` (csrc/wdb_sac_discrete.cu) compute the twin critics' and
the categorical actor's gradients of one TrainerDiscreteSAC update over the sampled windows of
the replay ring in place, and write them straight into the `.grad` views of the gradient arena.
alpha is read from log_alpha on the device.  The torch autograd update (algorithms/
sac_discrete.py) stays for the shapes these do not take."""
import ctypes

import torch

from warp_drive_b200 import lib as _lib
from warp_drive_b200.training.algorithms.fused_ddpg import _set_shape, replay_windows


def _layers(model):
    """[(weight, bias)] of the hidden Linear layers, then the head: the actor's one softmax head
    (policy_head[0]) or the Q network's policy_head."""
    head = model.policy_head
    if isinstance(head, torch.nn.ModuleList):
        head = head[0]
    return [(model.fc[str(i)][0].weight, model.fc[str(i)][0].bias)
            for i in range(len(model.fc))] + [(head.weight, head.bias)]


def _set_pointers(net, model, grads):
    for i, (w, b) in enumerate(_layers(model)):
        net.w[i], net.b[i] = _lib.ptr(w.data), _lib.ptr(b.data)
        if grads:
            net.gw[i], net.gb[i] = _lib.ptr(w.grad), _lib.ptr(b.grad)


def _shape_struct(actor, critic, n_envs, n_agents, capacity, n_step):
    u = _lib.SacDiscreteUpdate()
    u.n_envs, u.n_agents = int(n_envs), int(n_agents)
    u.obs_dim = int(actor.flattened_obs_size)
    u.n_actions = int(actor.output_dims[0])
    u.capacity, u.n_step = int(capacity), int(n_step)
    for net, model in ((u.actor, actor), (u.critic, critic), (u.critic2, critic),
                       (u.target_critic, critic), (u.target_critic2, critic)):
        _set_shape(net, model)
    return u


class FusedDiscreteSACUpdate:
    """One policy's two discrete SAC passes over `rows` sampled windows per update: the argument
    struct, one workspace for both (they run in order on one stream) and the loss sums (device
    double[4]: sum (Q1 - R)^2, sum (Q2 - R)^2, sum_g sum_a pi_a min(Q1, Q2)_a,
    sum_g sum_a pi_a log pi_a)."""

    @classmethod
    def supported(cls, actor, critic, critic2, n_envs, n_agents, capacity, n_step, rows):
        """True if both passes take this policy: TrainerDiscreteSAC's models (checked there) of
        0..3 hidden layers of width <= 64, both critics shaped alike, 2 <= A <= 64, F <= 63,
        and each pass's networks in one CTA's shared memory ([64, 64] fits both passes)."""
        if [int(w) for w in critic2.fc_dims] != [int(w) for w in critic.fc_dims]:
            return False
        u = _shape_struct(actor, critic, n_envs, n_agents, capacity, n_step)
        lib = _lib.load()
        return bool(lib.wdb_sac_discrete_critic_update_sampled_supported(ctypes.byref(u), rows)
                    and lib.wdb_sac_discrete_actor_update_sampled_supported(ctypes.byref(u), rows))

    def __init__(self, actor, critic, critic2, target_critic, target_critic2, log_alpha, n_envs,
                 n_agents, capacity, n_step, gamma, rows):
        self.models = (actor, critic, critic2, target_critic, target_critic2)
        self.log_alpha = log_alpha
        u = self.u = _shape_struct(actor, critic, n_envs, n_agents, capacity, n_step)
        u.gamma = float(gamma)
        self.lib = _lib.load()
        self.rows = int(rows)
        nbytes = max(
            int(self.lib.wdb_sac_discrete_critic_update_sampled_workspace_bytes(
                ctypes.byref(u), self.rows)),
            int(self.lib.wdb_sac_discrete_actor_update_sampled_workspace_bytes(
                ctypes.byref(u), self.rows)))
        assert nbytes > 0, "shapes not supported by wdb_sac_discrete_*_update_sampled"
        dev = next(actor.parameters()).device
        self.workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        self.sums = torch.zeros(4, dtype=torch.float64, device=dev)

    def _launch(self, name, obs, windows):
        u = self.u
        assert windows.shape[0] == self.rows
        u.obs = _lib.ptr(obs)
        u.log_alpha = _lib.ptr(self.log_alpha.data)
        u.sums = _lib.ptr(self.sums)
        u.workspace = _lib.ptr(self.workspace)
        rc = getattr(self.lib, f"wdb_{name}")(_lib.stream_ptr(), ctypes.byref(u),
                                             ctypes.byref(replay_windows(windows)))
        _lib.check(rc, name)
        return self.sums

    def critic_launch(self, obs, actions, rewards, done, windows, outputs=None):
        """Both critics' gradients into their `.grad`.  obs [C, E, Np, F], int32 actions
        [C, E, Np, 1], rewards [C, E, Np], done [C, E]: the ring in physical slot order; windows
        int32 [rows, 2].  outputs: optional (q1_values, q2_values, returns) tensors [rows]."""
        u = self.u
        actor, critic, critic2, target_critic, target_critic2 = self.models
        # parameters may have been re-allocated (load_state_dict keeps storage; .to() does not)
        _set_pointers(u.actor, actor, False)
        _set_pointers(u.critic, critic, True)
        _set_pointers(u.critic2, critic2, True)
        _set_pointers(u.target_critic, target_critic, False)
        _set_pointers(u.target_critic2, target_critic2, False)
        u.actions, u.rewards, u.done = _lib.ptr(actions), _lib.ptr(rewards), _lib.ptr(done)
        q1, q2, returns = outputs if outputs is not None else (None, None, None)
        u.q1_values, u.q2_values, u.returns = _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(returns)
        return self._launch("sac_discrete_critic_update_sampled", obs, windows)

    def actor_launch(self, obs, windows, entropies=None):
        """The actor's gradient into its `.grad`, through both critics as they are now.
        entropies: optional [rows] output."""
        u = self.u
        actor, critic, critic2 = self.models[:3]
        _set_pointers(u.actor, actor, True)
        _set_pointers(u.critic, critic, False)
        _set_pointers(u.critic2, critic2, False)
        u.entropies = _lib.ptr(entropies)
        return self._launch("sac_discrete_actor_update_sampled", obs, windows)
