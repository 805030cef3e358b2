"""Fused TQC update: `wdb_tqc_critic_update_sampled` and `wdb_tqc_actor_update_sampled`
(csrc/wdb_tqc.cu) compute the two quantile critics' and the squashed-Gaussian actor's gradients
of one TrainerTQC update over the sampled windows of the replay ring in place, and write them
straight into the `.grad` views of the gradient arena.  alpha is read from log_alpha on the
device.  The torch autograd update (algorithms/tqc.py) stays for the shapes these do not take:
M != 2 critics, or networks outside the passes' envelope."""
import ctypes

import torch

from warp_drive_b200 import lib as _lib
from warp_drive_b200.training.algorithms.fused_ddpg import (_set_pointers, _set_shape,
                                                            replay_windows)


def _shape_struct(actor, critic, n_envs, n_agents, capacity, n_step, n_drop):
    u = _lib.TqcUpdate()
    u.n_envs, u.n_agents = int(n_envs), int(n_agents)
    u.obs_dim = int(actor.flattened_obs_size)
    u.action_dim = int(actor.output_dims[0])
    u.capacity, u.n_step = int(capacity), int(n_step)
    u.n_quantiles, u.n_drop = int(critic.num_quantiles), int(n_drop)
    u.log_std_min, u.log_std_max = float(actor.log_std_min), float(actor.log_std_max)
    for net, model in ((u.actor, actor), (u.critic, critic), (u.critic2, critic),
                       (u.target_critic, critic), (u.target_critic2, critic)):
        _set_shape(net, model)
    return u


class FusedTQCUpdate:
    """One policy's two TQC passes over `rows` sampled windows per update: the argument struct,
    one workspace for both (they run in order on one stream) and the loss sums (device
    double[4]: sum_g loss_g, sum_g mean theta, sum_g Qbar_g, sum_g log pi)."""

    @classmethod
    def supported(cls, algo, actor, critics, n_envs, n_agents, capacity, n_step, rows):
        """True if both passes take this policy: TrainerTQC's models (checked there) with M = 2
        critics of one shape, 0..3 hidden layers of width <= 64 per network, 2N <= 64, A <= 32,
        F + A <= 64, and each pass's networks and tiles in one CTA's shared memory (the run
        config's [64, 64] networks with N = 25 fit)."""
        if algo.n_critics != 2 or len(critics) != 2:
            return False
        c1, c2 = critics[0], critics[1]
        if [int(w) for w in c2.fc_dims] != [int(w) for w in c1.fc_dims]:
            return False
        if not c1.num_quantiles == c2.num_quantiles == algo.n_quantiles:
            return False
        u = _shape_struct(actor, c1, n_envs, n_agents, capacity, n_step, algo.drop_per_net)
        lib = _lib.load()
        return bool(lib.wdb_tqc_critic_update_sampled_supported(ctypes.byref(u), rows)
                    and lib.wdb_tqc_actor_update_sampled_supported(ctypes.byref(u), rows))

    def __init__(self, algo, actor, critics, target_critics, log_alpha, n_envs, n_agents,
                 capacity, n_step, rows):
        self.models = (actor, critics[0], critics[1], target_critics[0], target_critics[1])
        self.log_alpha = log_alpha
        u = self.u = _shape_struct(actor, critics[0], n_envs, n_agents, capacity, n_step,
                                   algo.drop_per_net)
        u.gamma = float(algo.discount_factor_gamma)
        u.action_scale, u.action_bias = float(actor.action_scale), float(actor.action_bias)
        self.lib = _lib.load()
        self.rows = int(rows)
        self.kept_atoms = algo.kept_atoms
        nbytes = max(
            int(self.lib.wdb_tqc_critic_update_sampled_workspace_bytes(ctypes.byref(u),
                                                                       self.rows)),
            int(self.lib.wdb_tqc_actor_update_sampled_workspace_bytes(ctypes.byref(u),
                                                                      self.rows)))
        assert nbytes > 0, "shapes not supported by wdb_tqc_*_update_sampled"
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

    def critic_launch(self, obs, actions, rewards, done, noise, windows, outputs=None):
        """Both critics' gradients into their `.grad`.  obs [C, E, Np, F], actions [C, E, Np,
        A], rewards [C, E, Np], done [C, E]: the ring in physical slot order; noise [rows, A]
        standard normal (eps'); windows int32 [rows, 2].  outputs: optional (q_means,
        target_means) tensors [rows]."""
        u = self.u
        actor, critic, critic2, target_critic, target_critic2 = self.models
        # parameters may have been re-allocated (load_state_dict keeps storage; .to() does not)
        _set_pointers(u.actor, actor, False)
        _set_pointers(u.critic, critic, True)
        _set_pointers(u.critic2, critic2, True)
        _set_pointers(u.target_critic, target_critic, False)
        _set_pointers(u.target_critic2, target_critic2, False)
        u.actions, u.rewards, u.done = _lib.ptr(actions), _lib.ptr(rewards), _lib.ptr(done)
        u.critic_noise = _lib.ptr(noise)
        q_means, target_means = outputs if outputs is not None else (None, None)
        u.q_means, u.target_means = _lib.ptr(q_means), _lib.ptr(target_means)
        return self._launch("tqc_critic_update_sampled", obs, windows)

    def actor_launch(self, obs, noise, windows, log_probs=None):
        """The actor's gradient into its `.grad`, through both critics as they are now; noise
        [rows, A] (eps).  log_probs: optional [rows] output."""
        u = self.u
        actor, critic, critic2 = self.models[:3]
        _set_pointers(u.actor, actor, True)
        _set_pointers(u.critic, critic, False)
        _set_pointers(u.critic2, critic2, False)
        u.actor_noise = _lib.ptr(noise)
        u.log_probs = _lib.ptr(log_probs)
        return self._launch("tqc_actor_update_sampled", obs, windows)
