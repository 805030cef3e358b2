"""Fused DQN update: `wdb_dqn_update_sampled` (csrc/wdb_ddpg_update.cu) computes the Q
network's gradient of one TrainerDQN update over the sampled windows of the replay ring in
place -- the online and target forwards, the double-Q bootstrap, the n-step returns, the Huber
loss and the backward pass -- and writes it straight into the `.grad` views of the gradient
arena.  `wdb_qr_dqn_update_sampled` does the same for quantile-regression DQN
(FusedQRDQNUpdate).  The torch autograd updates (algorithms/dqn.py) stay for the shapes these do
not take."""
import ctypes

import torch

from warp_drive_b200 import lib as _lib
from warp_drive_b200.training.algorithms.fused_ddpg import (
    _set_pointers, _set_shape, replay_windows)
from warp_drive_b200.utils.spaces import Box


def _shape_struct(algo, q_net, n_envs, n_agents, capacity):
    u = _lib.DqnUpdate()
    u.n_envs, u.n_agents = int(n_envs), int(n_agents)
    u.obs_dim, u.n_actions = int(q_net.flattened_obs_size), int(q_net.output_dims[0])
    u.capacity, u.n_step = int(capacity), int(algo.n_step)
    u.gamma, u.huber_delta = float(algo.discount_factor_gamma), float(algo.huber_delta)
    u.double_q = int(algo.double_q)
    _set_shape(u.q, q_net)
    _set_shape(u.target_q, q_net)
    return u


def fused_dqn_supported(algo, q_net, n_envs, n_agents, capacity, replay_rows):
    """True if `wdb_dqn_update_sampled` takes this policy: a FullyConnectedQ over a Box
    observation with 0..3 hidden layers of width <= 64, A <= 64 and F <= 63, and replay_rows
    sampled windows per update."""
    from warp_drive_b200.training.models.fully_connected_q import FullyConnectedQ

    if type(q_net) is not FullyConnectedQ or not isinstance(q_net.observation_space, Box):
        return False
    if len(q_net.fc_dims) > 3:
        return False
    u = _shape_struct(algo, q_net, n_envs, n_agents, capacity)
    return bool(_lib.load().wdb_dqn_update_sampled_supported(ctypes.byref(u), int(replay_rows)))


class FusedDQNUpdate:
    """One policy's `wdb_dqn_update_sampled` launch: the argument struct, its workspace and the
    loss sums (device double[2]: sum huber(Q - R), sum Q(obs, a))."""

    def __init__(self, algo, q_net, target_net, n_envs, n_agents, capacity, replay_rows):
        self.models = (q_net, target_net)
        self.u = _shape_struct(algo, q_net, n_envs, n_agents, capacity)
        self.lib = _lib.load()
        self.rows = int(replay_rows)
        nbytes = int(self.lib.wdb_dqn_update_sampled_workspace_bytes(
            ctypes.byref(self.u), self.rows))
        assert nbytes > 0, "shapes not supported by wdb_dqn_update_sampled"
        dev = next(q_net.parameters()).device
        self.workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        self.sums = torch.zeros(2, dtype=torch.float64, device=dev)

    def launch(self, obs, actions, rewards, done, windows, outputs=None, weights=None):
        """The Q network's gradient into its `.grad`.  obs [C, E, Np, F], actions [C, E, Np, 1]
        (int32), rewards [C, E, Np], done [C, E] are the ring in physical slot order; windows
        int32 [rows, 2] the sampled windows.  outputs: optional (q_values, returns) float32
        tensors [rows] for the metrics.  weights: float32 [rows] importance-sampling weights
        (prioritized replay): wdb_dqn_update_prioritized instead of wdb_dqn_update_sampled."""
        u = self.u
        q_net, target_net = self.models
        # parameters may have been re-allocated (load_state_dict keeps storage; .to() does not)
        _set_pointers(u.q, q_net, True)
        _set_pointers(u.target_q, target_net, False)
        u.obs, u.actions = _lib.ptr(obs), _lib.ptr(actions)
        u.rewards, u.done = _lib.ptr(rewards), _lib.ptr(done)
        q_values, returns = outputs if outputs is not None else (None, None)
        u.q_values, u.returns = _lib.ptr(q_values), _lib.ptr(returns)
        u.sums = _lib.ptr(self.sums)
        u.workspace = _lib.ptr(self.workspace)
        assert windows.shape[0] == self.rows
        if weights is None:
            _lib.check(self.lib.wdb_dqn_update_sampled(
                _lib.stream_ptr(), ctypes.byref(u), ctypes.byref(replay_windows(windows))),
                "dqn_update_sampled")
        else:
            assert weights.shape == (self.rows,) and weights.dtype == torch.float32
            _lib.check(self.lib.wdb_dqn_update_prioritized(
                _lib.stream_ptr(), ctypes.byref(u), ctypes.byref(replay_windows(windows)),
                _lib.ptr(weights)), "dqn_update_prioritized")
        return self.sums


def fused_qr_dqn_supported(algo, q_net, n_envs, n_agents, capacity, replay_rows):
    """True if `wdb_qr_dqn_update_sampled` takes this policy: a FullyConnectedQuantileQ over a
    Box observation with 0..3 hidden layers of width <= 64, F <= 63 and a head of
    A * num_quantiles <= 64 outputs, and replay_rows sampled windows per update."""
    from warp_drive_b200.training.models.fully_connected_q import FullyConnectedQuantileQ

    if type(q_net) is not FullyConnectedQuantileQ or not isinstance(q_net.observation_space,
                                                                    Box):
        return False
    if len(q_net.fc_dims) > 3:
        return False
    u = _shape_struct(algo, q_net, n_envs, n_agents, capacity)
    return bool(_lib.load().wdb_qr_dqn_update_sampled_supported(
        ctypes.byref(u), int(q_net.num_quantiles), int(replay_rows)))


class FusedQRDQNUpdate:
    """One policy's `wdb_qr_dqn_update_sampled` launch: DQN's argument struct with the number
    of quantiles beside it; the sums are sum w_g loss_g and sum Q-bar, the outputs Q-bar and
    R-bar."""

    def __init__(self, algo, q_net, target_net, n_envs, n_agents, capacity, replay_rows):
        self.models = (q_net, target_net)
        self.u = _shape_struct(algo, q_net, n_envs, n_agents, capacity)
        self.n_quantiles = int(q_net.num_quantiles)
        self.lib = _lib.load()
        self.rows = int(replay_rows)
        nbytes = int(self.lib.wdb_qr_dqn_update_sampled_workspace_bytes(
            ctypes.byref(self.u), self.n_quantiles, self.rows))
        assert nbytes > 0, "shapes not supported by wdb_qr_dqn_update_sampled"
        dev = next(q_net.parameters()).device
        self.workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        self.sums = torch.zeros(2, dtype=torch.float64, device=dev)

    def launch(self, obs, actions, rewards, done, windows, outputs=None, weights=None):
        """The quantile network's gradient into its `.grad`; the arguments of
        FusedDQNUpdate.launch (outputs: Q-bar and R-bar)."""
        u = self.u
        q_net, target_net = self.models
        _set_pointers(u.q, q_net, True)
        _set_pointers(u.target_q, target_net, False)
        u.obs, u.actions = _lib.ptr(obs), _lib.ptr(actions)
        u.rewards, u.done = _lib.ptr(rewards), _lib.ptr(done)
        q_values, returns = outputs if outputs is not None else (None, None)
        u.q_values, u.returns = _lib.ptr(q_values), _lib.ptr(returns)
        u.sums = _lib.ptr(self.sums)
        u.workspace = _lib.ptr(self.workspace)
        assert windows.shape[0] == self.rows
        if weights is not None:
            assert weights.shape == (self.rows,) and weights.dtype == torch.float32
        _lib.check(self.lib.wdb_qr_dqn_update_sampled(
            _lib.stream_ptr(), ctypes.byref(u), self.n_quantiles,
            ctypes.byref(replay_windows(windows)), _lib.ptr(weights)), "qr_dqn_update_sampled")
        return self.sums
