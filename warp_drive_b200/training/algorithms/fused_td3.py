"""Fused TD3 update: `wdb_td3_critic_update` and `wdb_td3_actor_update`
(csrc/wdb_ddpg_update.cu) compute the twin critics' and the actor's gradients of one TrainerTD3
update from the replay ring in place, on the tile primitives of the fused DDPG update, and
write them straight into the `.grad` views of the gradient arena.  The torch autograd update
(algorithms/td3.py) stays for the shapes these do not take."""
import ctypes

import torch

from warp_drive_b200 import lib as _lib
from warp_drive_b200.training.algorithms.fused_ddpg import (_set_pointers, _set_shape,
                                                            fused_models_supported,
                                                            replay_windows)


def _shape_struct(algo, actor, critic, n_envs, n_agents, capacity, n_step):
    u = _lib.Td3Update()
    u.n_envs, u.n_agents = int(n_envs), int(n_agents)
    u.obs_dim = int(actor.flattened_obs_size)
    u.action_dim = int(actor.output_dims[0])
    u.capacity, u.cursor, u.n_step = int(capacity), 0, int(n_step)
    u.target_noise, u.target_noise_clip = algo.target_noise, algo.target_noise_clip
    for net, model in ((u.actor, actor), (u.critic, critic), (u.critic2, critic),
                       (u.target_actor, actor), (u.target_critic, critic),
                       (u.target_critic2, critic)):
        _set_shape(net, model)
    return u


def fused_td3_supported(algo, actor, critic, critic2, n_envs, n_agents, capacity, n_step,
                        replay_rows=None):
    """True if both TD3 passes take this policy: the networks `fused_ddpg_supported` takes,
    two critics of one shape, and five networks plus two critic gradient blocks in one CTA's
    shared memory (0..3 hidden layers; [64, 64] fits, three layers of 64 do not)."""
    if critic2 is None or [int(w) for w in critic2.fc_dims] != [int(w) for w in critic.fc_dims]:
        return False
    if type(critic2) is not type(critic) or critic2.flattened_obs_size != critic.flattened_obs_size:
        return False
    if not fused_models_supported(algo, actor, critic):
        return False
    u = _shape_struct(algo, actor, critic, n_envs, n_agents, capacity, n_step)
    lib = _lib.load()
    if replay_rows is not None:     # the passes over that many sampled windows per update
        return bool(lib.wdb_td3_critic_update_sampled_supported(ctypes.byref(u), replay_rows)
                    and lib.wdb_td3_actor_update_sampled_supported(ctypes.byref(u), replay_rows))
    return bool(lib.wdb_td3_critic_update_supported(ctypes.byref(u))
                and lib.wdb_td3_actor_update_supported(ctypes.byref(u)))


class FusedTD3Update:
    """One policy's two TD3 passes: the argument struct, one workspace for both (they run in
    order on one stream) and the loss sums (device double[4]: sum (Q1 - R)^2, sum (Q2 - R)^2,
    sum J, 0)."""

    def __init__(self, algo, actor, critic, critic2, target_actor, target_critic,
                 target_critic2, n_envs, n_agents, capacity, n_step, gamma, replay_rows=None):
        self.models = (actor, critic, critic2, target_actor, target_critic, target_critic2)
        u = self.u = _shape_struct(algo, actor, critic, n_envs, n_agents, capacity, n_step)
        u.gamma = float(gamma)
        u.action_scale, u.action_bias = float(actor.action_scale), float(actor.action_bias)
        self.lib = _lib.load()
        if replay_rows is None:
            nbytes = max(int(self.lib.wdb_td3_critic_update_workspace_bytes(ctypes.byref(u))),
                         int(self.lib.wdb_td3_actor_update_workspace_bytes(ctypes.byref(u))))
        else:
            nbytes = max(int(self.lib.wdb_td3_critic_update_sampled_workspace_bytes(
                ctypes.byref(u), replay_rows)), int(
                    self.lib.wdb_td3_actor_update_sampled_workspace_bytes(
                        ctypes.byref(u), replay_rows)))
        assert nbytes > 0, "shapes not supported by wdb_td3_*_update"
        dev = next(actor.parameters()).device
        self.workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        self.sums = torch.zeros(4, dtype=torch.float64, device=dev)
        self.valid = int(capacity) - int(n_step) + 1
        # loss rows per update: every window of the ring, or replay_rows sampled windows
        self.rows = self.valid * int(n_envs) * int(n_agents) if replay_rows is None else int(
            replay_rows)

    def _launch(self, name, windows):
        """Pass `name` over the ring, or over `windows` (int32 [rows, 2]: the _sampled pass;
        the cursor is not read, noise and outputs are per sampled row)."""
        if windows is None:
            rc = getattr(self.lib, f"wdb_{name}")(_lib.stream_ptr(), ctypes.byref(self.u))
        else:
            assert windows.shape[0] == self.rows
            rc = getattr(self.lib, f"wdb_{name}_sampled")(
                _lib.stream_ptr(), ctypes.byref(self.u), ctypes.byref(replay_windows(windows)))
        _lib.check(rc, name)

    def _ring(self, obs, cursor):
        u = self.u
        u.cursor = int(cursor)
        u.obs = _lib.ptr(obs)
        u.sums = _lib.ptr(self.sums)
        u.workspace = _lib.ptr(self.workspace)

    def critic_launch(self, obs, actions, rewards, done, cursor, noise, outputs=None,
                      windows=None):
        """Both critics' gradients into their `.grad`.  obs [C, E, Np, F], actions [C, E, Np,
        A], rewards [C, E, Np], done [C, E]: the ring in physical slot order, `cursor` its
        oldest slot; noise [valid, E, Np, A] standard normal in window order.  outputs:
        optional (q1_values, q2_values, returns) tensors [valid, E, Np]."""
        u = self.u
        _, critic, critic2, target_actor, target_critic, target_critic2 = self.models
        # parameters may have been re-allocated (load_state_dict keeps storage; .to() does not)
        _set_pointers(u.critic, critic, True)
        _set_pointers(u.critic2, critic2, True)
        _set_pointers(u.target_actor, target_actor, False)
        _set_pointers(u.target_critic, target_critic, False)
        _set_pointers(u.target_critic2, target_critic2, False)
        self._ring(obs, cursor)
        u.actions, u.rewards, u.done = _lib.ptr(actions), _lib.ptr(rewards), _lib.ptr(done)
        u.noise = _lib.ptr(noise)
        q1, q2, returns = outputs if outputs is not None else (None, None, None)
        u.q1_values, u.q2_values, u.returns = _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(returns)
        self._launch("td3_critic_update", windows)
        return self.sums

    def actor_launch(self, obs, cursor, j_values=None, windows=None):
        """The actor's gradient into its `.grad`, through the critic as it is now.  j_values:
        optional [valid, E, Np] output."""
        u = self.u
        actor, critic = self.models[:2]
        _set_pointers(u.actor, actor, True)
        _set_pointers(u.critic, critic, True)
        self._ring(obs, cursor)
        u.j_values = _lib.ptr(j_values)
        self._launch("td3_actor_update", windows)
        return self.sums
