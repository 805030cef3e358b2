"""Fused DQN update: `wdb_dqn_update_sampled` (csrc/wdb_ddpg_update.cu) computes the Q
network's gradient of one TrainerDQN update over the sampled windows of the replay ring in
place -- the online and target forwards, the double-Q bootstrap, the n-step returns, the Huber
loss and the backward pass -- and writes it straight into the `.grad` views of the gradient
arena.  `wdb_qr_dqn_update_sampled` does the same for quantile-regression DQN
(FusedQRDQNUpdate) and `wdb_iqn_update_sampled` (csrc/wdb_iqn_update.cu) for implicit quantile
networks (FusedIQNUpdate), and `wdb_c51_update_sampled` (csrc/wdb_c51_update.cu) for categorical
DQN (FusedC51Update).  A dueling DQN or C51 network runs the same passes on its folded network
(FusedDuelingUpdate; csrc/wdb_dueling.cu folds the head before the pass and unfolds its gradients
after it).  A noisy DQN or C51 network, plain or dueling, runs them on its materialized head
(FusedNoisyUpdate; csrc/wdb_noisy.cu draws the update's noise and writes the effective layers
before the pass, and maps their gradients onto mu and sigma after it).  The torch autograd
updates (algorithms/dqn.py) stay for the shapes these do not take.  An action-masked DQN or C51
network (plain, dueling or noisy) runs `wdb_dqn_update_masked` / `wdb_c51_update_masked`
(csrc/wdb_masked_q.cu; FusedMaskedDQNUpdate, FusedMaskedC51Update), whose bootstrap ranges over
the valid actions of obs' own mask; masked QR-DQN and IQN networks train through the torch
losses.  A branching network (one Q head per action dimension of a MultiDiscrete space) runs
`wdb_branching_dqn_update_sampled` (csrc/wdb_branching_q.cu; FusedBranchingDQNUpdate)."""
import ctypes

import torch

from warp_drive_b200 import lib as _lib
from warp_drive_b200.training.algorithms.fused_ddpg import (
    _set_pointers, _set_shape, replay_windows)
from warp_drive_b200.training.models.fully_connected_q import (
    FullyConnectedBranchingQ, FullyConnectedCategoricalQ, FullyConnectedIQN, FullyConnectedQ,
    FullyConnectedQuantileQ)
from warp_drive_b200.utils.spaces import Box


def _masked(q_net):
    """Whether a Q network's observations carry an action mask (FullyConnectedQ.masked)."""
    return bool(getattr(q_net, "masked", False))


def _shape_struct(algo, q_net, n_envs, n_agents, capacity):
    u = _lib.DqnUpdate()
    u.n_envs, u.n_agents = int(n_envs), int(n_agents)
    u.obs_dim, u.n_actions = int(q_net.flattened_obs_size), int(q_net.output_dims[0])
    if getattr(q_net, "is_branching_q", False):   # the heads side by side: A = sum_d A_d
        u.n_actions = int(sum(q_net.branch_sizes))
    u.capacity, u.n_step = int(capacity), int(algo.n_step)
    u.gamma, u.huber_delta = float(algo.discount_factor_gamma), float(algo.huber_delta)
    u.double_q = int(algo.double_q)
    _set_shape(u.q, q_net)
    _set_shape(u.target_q, q_net)
    return u


class FusedQUpdate:
    """One policy's launch of a Q network's replay pass `wdb_<entry>`: DQN's argument struct,
    the pass's workspace and the loss sums (device double[2]).  A pass names the model type it
    takes and its entry point, and states the arguments the entry takes between the struct and
    the windows (`shape_args` for `_supported` / `_workspace_bytes`, `launch_args` for the
    launch)."""
    model = None
    entry = None
    masked = False                             # the pass takes action-masked networks only

    @staticmethod
    def shape_args(q_net):
        return ()

    @classmethod
    def supported(cls, algo, q_net, n_envs, n_agents, capacity, replay_rows):
        """True if `wdb_<entry>` takes this policy: a `model` over a Box observation (a masked
        pass: an action-masked network, over its Dict observation) with at most 3 hidden layers,
        no dueling head (FusedDuelingUpdate) and no noisy head (FusedNoisyUpdate), in the pass's
        envelope for replay_rows sampled windows per update."""
        if type(q_net) is not cls.model or _masked(q_net) != cls.masked:
            return False
        if not cls.masked and not isinstance(q_net.observation_space, Box):
            return False
        if q_net.dueling or q_net.noisy or len(q_net.fc_dims) > 3:
            return False
        return cls.fits(_shape_struct(algo, q_net, n_envs, n_agents, capacity), q_net,
                        replay_rows)

    @classmethod
    def fits(cls, u, q_net, replay_rows):
        """`wdb_<entry>_supported` of the shape struct u."""
        return bool(getattr(_lib.load(), f"wdb_{cls.entry}_supported")(
            ctypes.byref(u), *cls.shape_args(q_net), int(replay_rows)))

    def __init__(self, algo, q_net, target_net, n_envs, n_agents, capacity, replay_rows, u=None,
                 point=None):
        """u and point stand in for q_net's shape struct and pointer step when the pass runs on
        another network of its shape (FusedDuelingUpdate: the trunk and the folded head)."""
        self.models = (q_net, target_net)
        self.u = _shape_struct(algo, q_net, n_envs, n_agents, capacity) if u is None else u
        self.point = self._point if point is None else point
        self.lib = _lib.load()
        self.rows = int(replay_rows)
        nbytes = int(getattr(self.lib, f"wdb_{self.entry}_workspace_bytes")(
            ctypes.byref(self.u), *self.shape_args(q_net), self.rows))
        assert nbytes > 0, f"shapes not supported by wdb_{self.entry}"
        dev = next(q_net.parameters()).device
        self.workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        self.sums = torch.zeros(2, dtype=torch.float64, device=dev)

    def _point(self, u):
        q_net, target_net = self.models
        _set_pointers(u.q, q_net, True)
        _set_pointers(u.target_q, target_net, False)

    def launch_args(self):
        return self.shape_args(self.models[0])

    def launch(self, obs, actions, rewards, done, windows, outputs=None, weights=None):
        """The Q network's gradient into its `.grad`.  obs [C, E, Np, F], actions [C, E, Np, 1]
        (int32), rewards [C, E, Np], done [C, E] are the ring in physical slot order; windows
        int32 [rows, 2] the sampled windows.  outputs: optional (q_values, returns) float32
        tensors [rows] for the metrics.  weights: float32 [rows] importance-sampling weights
        (prioritized replay)."""
        u = self.u
        # parameters may have been re-allocated (load_state_dict keeps storage; .to() does not)
        self.point(u)
        u.obs, u.actions = _lib.ptr(obs), _lib.ptr(actions)
        u.rewards, u.done = _lib.ptr(rewards), _lib.ptr(done)
        q_values, returns = outputs if outputs is not None else (None, None)
        u.q_values, u.returns = _lib.ptr(q_values), _lib.ptr(returns)
        u.sums = _lib.ptr(self.sums)
        u.workspace = _lib.ptr(self.workspace)
        assert windows.shape[0] == self.rows
        if weights is not None:
            assert weights.shape == (self.rows,) and weights.dtype == torch.float32
        self._run(ctypes.byref(u), ctypes.byref(replay_windows(windows)), weights)
        return self.sums

    def _run(self, u, windows, weights):
        _lib.check(getattr(self.lib, f"wdb_{self.entry}")(
            _lib.stream_ptr(), u, *self.launch_args(), windows, _lib.ptr(weights)), self.entry)


class FusedDQNUpdate(FusedQUpdate):
    """`wdb_dqn_update_sampled` (FullyConnectedQ): 0..3 hidden layers of width <= 64, A <= 64 and
    F <= 63.  The sums are sum huber(Q - R) and sum Q(obs, a).  With weights the launch is
    `wdb_dqn_update_prioritized`, which takes the same shapes and workspace."""
    model = FullyConnectedQ
    entry = "dqn_update_sampled"

    def _run(self, u, windows, weights):
        if weights is None:
            _lib.check(self.lib.wdb_dqn_update_sampled(_lib.stream_ptr(), u, windows),
                       "dqn_update_sampled")
        else:
            _lib.check(self.lib.wdb_dqn_update_prioritized(
                _lib.stream_ptr(), u, windows, _lib.ptr(weights)), "dqn_update_prioritized")


def q_branches(q_net):
    """struct wdb_q_branches of a FullyConnectedBranchingQ, or None when it has more heads than
    the struct holds (such a network trains through the torch loss)."""
    sizes = q_net.branch_sizes
    if len(sizes) > _lib.Q_MAX_BRANCHES:
        return None
    b = _lib.QBranches()
    b.n_heads = len(sizes)
    for d, a in enumerate(sizes):
        b.sizes[d] = int(a)
    return b


class FusedBranchingDQNUpdate(FusedQUpdate):
    """`wdb_branching_dqn_update_sampled` (FullyConnectedBranchingQ): DQN's shapes with the head
    A = sum_d A_d <= 64 and 1 <= D <= 16 heads, the heads' sizes beside the struct; actions
    [C, E, Np, D].  The sums are sum_g w_g (1/D) sum_d huber(Q_d - R) and sum Q-bar, the outputs
    Q-bar and R.  With weights the launch is `wdb_branching_dqn_update_prioritized`, which takes
    the same shapes and workspace."""
    model = FullyConnectedBranchingQ
    entry = "branching_dqn_update_sampled"

    @staticmethod
    def shape_args(q_net):
        return (ctypes.byref(q_branches(q_net)),)

    @classmethod
    def fits(cls, u, q_net, replay_rows):
        return q_branches(q_net) is not None and super().fits(u, q_net, replay_rows)

    def __init__(self, algo, q_net, *args, **kwargs):
        super().__init__(algo, q_net, *args, **kwargs)
        self.branches = q_branches(q_net)

    def _run(self, u, windows, weights):
        if weights is None:
            _lib.check(self.lib.wdb_branching_dqn_update_sampled(
                _lib.stream_ptr(), u, ctypes.byref(self.branches), windows),
                "branching_dqn_update_sampled")
        else:
            _lib.check(self.lib.wdb_branching_dqn_update_prioritized(
                _lib.stream_ptr(), u, ctypes.byref(self.branches), windows, _lib.ptr(weights)),
                "branching_dqn_update_prioritized")


class FusedQRDQNUpdate(FusedQUpdate):
    """`wdb_qr_dqn_update_sampled` (FullyConnectedQuantileQ): DQN's shapes with a head of
    A * num_quantiles <= 64 outputs, the number of quantiles beside the struct.  The sums are
    sum w_g loss_g and sum Q-bar, the outputs Q-bar and R-bar."""
    model = FullyConnectedQuantileQ
    entry = "qr_dqn_update_sampled"

    @staticmethod
    def shape_args(q_net):
        return (int(q_net.num_quantiles),)


def _iqn_struct(q_net, target_net=None):
    """struct wdb_iqn_args of an IQN pair: the counts, and the embeddings' pointers when the
    networks are given."""
    a = _lib.IqnArgs()
    a.n_cos, a.n_tau = int(q_net.num_cosines), int(q_net.num_tau_samples)
    a.n_tau_prime = int(q_net.num_tau_prime_samples)
    a.n_quantile_samples = int(q_net.num_quantile_samples)
    if target_net is not None:
        for net, model, grads in ((a.embed, q_net, True), (a.target_embed, target_net, False)):
            e = model.tau_embedding
            net.w[0], net.b[0] = _lib.ptr(e.weight.data), _lib.ptr(e.bias.data)
            if grads:
                net.gw[0], net.gb[0] = _lib.ptr(e.weight.grad), _lib.ptr(e.bias.grad)
    return a


class FusedIQNUpdate(FusedQUpdate):
    """`wdb_iqn_update_sampled` (FullyConnectedIQN): DQN's shapes with 1..3 hidden layers, n_cos,
    N and N' <= 64, everything in one CTA's shared memory, and the IQN struct beside DQN's.  The
    sums are sum w_g loss_g and sum Q-bar, the outputs Q-bar and R-bar."""
    model = FullyConnectedIQN
    entry = "iqn_update_sampled"

    @staticmethod
    def shape_args(q_net):
        return (ctypes.byref(_iqn_struct(q_net)),)

    def launch_args(self):
        return (ctypes.byref(self.iqn),)

    def launch(self, obs, actions, rewards, done, windows, outputs=None, weights=None,
               taus=None):
        """The network's gradient (trunk, head and tau embedding) into its `.grad`; the
        arguments of FusedQUpdate.launch and the levels `taus`, float32 [rows, N + N']."""
        iqn = self.iqn = _iqn_struct(*self.models)
        n = iqn.n_tau + iqn.n_tau_prime
        assert taus is not None and taus.shape == (self.rows, n) and taus.dtype == torch.float32
        assert taus.is_contiguous()
        iqn.taus = _lib.ptr(taus)
        return super().launch(obs, actions, rewards, done, windows, outputs, weights)


class FusedC51Update(FusedQUpdate):
    """`wdb_c51_update_sampled` (FullyConnectedCategoricalQ): DQN's shapes with 2 <= N <= 64
    atoms and everything in one CTA's shared memory; the number of atoms, the model's support
    (float32, on the device) and its spacing beside the struct.  The sums are sum w_g loss_g
    and sum Q-bar, the outputs Q-bar and R-bar."""
    model = FullyConnectedCategoricalQ
    entry = "c51_update_sampled"

    @staticmethod
    def shape_args(q_net):
        return (int(q_net.num_atoms),)

    def __init__(self, algo, q_net, *args, **kwargs):
        super().__init__(algo, q_net, *args, **kwargs)
        self.support = q_net.support.to(device=self.sums.device,
                                        dtype=torch.float32).contiguous()
        self.delta_z = float(q_net.delta_z)

    def launch_args(self):
        return self.shape_args(self.models[0]) + (_lib.ptr(self.support), self.delta_z)


class _MaskedQPass:
    """The action-masked form of a Q pass: `launch` also takes `action_mask`, the ring's mask
    array float32 [C, E, Np, A] (action_mask_batch_{p}), and `wdb_<entry>` takes it after the
    windows and the weights.  The bootstrap's a* ranges over the valid actions of obs' own mask
    row; the struct, workspace, sums and outputs are the unmasked pass's."""
    masked = True

    def launch(self, obs, actions, rewards, done, windows, outputs=None, weights=None,
               action_mask=None):
        assert action_mask is not None and action_mask.dtype == torch.float32
        assert action_mask.is_contiguous()
        assert tuple(action_mask.shape) == tuple(actions.shape[:-1]) + (self.u.n_actions,)
        self.action_mask = action_mask
        return super().launch(obs, actions, rewards, done, windows, outputs, weights)

    def _run(self, u, windows, weights):
        _lib.check(getattr(self.lib, f"wdb_{self.entry}")(
            _lib.stream_ptr(), u, *self.launch_args(), windows, _lib.ptr(weights),
            _lib.ptr(self.action_mask)), self.entry)


class FusedMaskedDQNUpdate(_MaskedQPass, FusedDQNUpdate):
    """`wdb_dqn_update_masked` (an action-masked FullyConnectedQ): FusedDQNUpdate's shapes, sums
    and outputs, uniform or weighted, with the masked bootstrap."""
    entry = "dqn_update_masked"


class FusedMaskedC51Update(_MaskedQPass, FusedC51Update):
    """`wdb_c51_update_masked` (an action-masked FullyConnectedCategoricalQ): FusedC51Update's
    shapes, sums and outputs, uniform or weighted, with the masked a*."""
    entry = "c51_update_masked"


def _mask_kwargs(action_mask):
    """The `action_mask` keyword of a plain pass's launch: only for a masked one."""
    return {} if action_mask is None else {"action_mask": action_mask}


def folded_widths(q_net):
    """The hidden widths of a dueling network's folded form: the trunk's, then the stacked
    stream hidden layer 2S when S > 0 (DuelingHead.folded)."""
    s = q_net.policy_head.stream_dim
    return [int(w) for w in q_net.fc_dims] + ([2 * s] if s else [])


def dueling_shape(head):
    """struct wdb_dueling_head of a DuelingHead with its shape only (no pointers)."""
    d = _lib.DuelingHead()
    d.n_actions, d.n_atoms = int(head.n_actions), int(head.n_outputs)
    d.in_dim, d.stream_dim = int(head.in_features), int(head.stream_dim)
    return d


def _live_stream(layer):
    """(weight, bias, weight grad, bias grad) of a plain stream Linear."""
    return layer.weight.data, layer.bias.data, layer.weight.grad, layer.bias.grad


class DuelingFold:
    """A DuelingHead's folded layers in buffers of their own (and, with grads, buffers for their
    gradients), and the struct wdb_dueling_head that ties them to the live stream parameters --
    or, given `source` (a stream layer -> its (weight, bias, weight grad, bias grad)), to other
    tensors of the streams' shapes (FusedNoisyUpdate: the materialized noisy layers)."""

    def __init__(self, model, grads=False, source=_live_stream):
        self.model, self.source = model, source
        head = model.policy_head
        s, h, out = head.stream_dim, head.in_features, head.out_features
        shapes = ([(2 * s, h), (2 * s,)] if s else []) + [(out, 2 * s if s else h), (out,)]
        dev = next(model.parameters()).device

        def buffers():
            t = [torch.zeros(shape, dtype=torch.float32, device=dev) for shape in shapes]
            return list(zip(t[0::2], t[1::2]))
        self.layers = buffers()                  # [(weight, bias)]: [hidden,] output
        self.grads = buffers() if grads else None

    def struct(self):
        head = self.model.policy_head
        d = dueling_shape(head)
        (vh, vo), (ah, ao) = head.streams()
        for prefix, hidden, out in (("value_", vh, vo), ("adv_", ah, ao)):
            for name, layer in (("h", hidden), ("o", out)):
                if layer is None:
                    continue
                w, b, gw, gb = self.source(layer)
                setattr(d, prefix + name + "w", _lib.ptr(w))
                setattr(d, prefix + name + "b", _lib.ptr(b))
                if self.grads is not None:
                    setattr(d, prefix + "g" + name + "w", _lib.ptr(gw))
                    setattr(d, prefix + "g" + name + "b", _lib.ptr(gb))
        names = (["h"] if head.stream_dim else []) + ["o"]
        for name, (w, b) in zip(names, self.layers):
            setattr(d, name + "w", _lib.ptr(w))
            setattr(d, name + "b", _lib.ptr(b))
        for name, (w, b) in zip(names, self.grads or []):
            setattr(d, "g" + name + "w", _lib.ptr(w))
            setattr(d, "g" + name + "b", _lib.ptr(b))
        return d


def fold(online, target=None):
    """wdb_dueling_fold of one or two DuelingFolds: one launch."""
    t = None if target is None else ctypes.byref(target.struct())
    _lib.check(_lib.load().wdb_dueling_fold(_lib.stream_ptr(), ctypes.byref(online.struct()), t),
               "dueling_fold")


def _dueling_shape_struct(algo, q_net, n_envs, n_agents, capacity):
    """_shape_struct with the folded network's hidden widths."""
    u = _shape_struct(algo, q_net, n_envs, n_agents, capacity)
    widths = folded_widths(q_net)
    for net in (u.q, u.target_q):
        net.n_hidden = len(widths)
        for i, w in enumerate(widths):
            net.widths[i] = w
    return u


class FusedDuelingUpdate:
    """One update of a dueling DQN or C51 policy: wdb_dueling_fold of the online and the target
    head (1 launch), the plain pass -- FusedDQNUpdate or FusedC51Update -- on networks made of the
    live trunk layers and the folded layers (2 launches), then wdb_dueling_unfold_grads (1
    launch).  The pass writes the trunk's gradients straight into the arena's `.grad` views and
    the folded layers' into scratch, which the unfold maps onto the stream parameters' `.grad`
    views.  Sums and outputs are the plain pass's."""

    @staticmethod
    def plain_type(q_net):
        categorical = getattr(q_net, "is_categorical_q", False)
        if _masked(q_net):
            return FusedMaskedC51Update if categorical else FusedMaskedDQNUpdate
        return FusedC51Update if categorical else FusedDQNUpdate

    @classmethod
    def supported(cls, algo, q_net, n_envs, n_agents, capacity, replay_rows):
        """True if the folded network of a dueling FullyConnectedQ or FullyConnectedCategoricalQ
        is in the plain pass's envelope: at most 3 hidden layers in all (a one-layer stream
        allows a trunk of at most 2), each, 2S included, of width <= 64, F <= 63, and C51's
        shared-memory cap."""
        if type(q_net) not in (FullyConnectedQ, FullyConnectedCategoricalQ) or not q_net.dueling:
            return False
        if q_net.noisy:                        # FusedNoisyUpdate
            return False
        if not (_masked(q_net) or isinstance(q_net.observation_space, Box)):
            return False
        if len(folded_widths(q_net)) > 3:
            return False
        head = ctypes.byref(dueling_shape(q_net.policy_head))
        if not _lib.load().wdb_dueling_fold_supported(head):
            return False
        u = _dueling_shape_struct(algo, q_net, n_envs, n_agents, capacity)
        return cls.plain_type(q_net).fits(u, q_net, replay_rows)

    def __init__(self, algo, q_net, target_net, n_envs, n_agents, capacity, replay_rows):
        self.online, self.target = DuelingFold(q_net, grads=True), DuelingFold(target_net)
        self.plain = self.plain_type(q_net)(
            algo, q_net, target_net, n_envs, n_agents, capacity, replay_rows,
            u=_dueling_shape_struct(algo, q_net, n_envs, n_agents, capacity), point=self._point)
        self.rows, self.sums = self.plain.rows, self.plain.sums

    def _point(self, u):
        for net, folded, grads in ((u.q, self.online, True), (u.target_q, self.target, False)):
            fc = folded.model.fc
            trunk = [(fc[str(i)][0].weight, fc[str(i)][0].bias) for i in range(len(fc))]
            for i, (w, b) in enumerate(trunk + folded.layers):
                net.w[i], net.b[i] = _lib.ptr(w.data), _lib.ptr(b.data)
            if grads:
                for i, (w, b) in enumerate([(w.grad, b.grad) for w, b in trunk] + folded.grads):
                    net.gw[i], net.gb[i] = _lib.ptr(w), _lib.ptr(b)

    def launch(self, obs, actions, rewards, done, windows, outputs=None, weights=None,
               action_mask=None):
        """The network's gradient (trunk and both streams) into its `.grad`; the arguments of
        FusedQUpdate.launch, and a masked network's `action_mask` for its masked pass."""
        fold(self.online, self.target)
        self.plain.launch(obs, actions, rewards, done, windows, outputs, weights,
                          **_mask_kwargs(action_mask))
        _lib.check(_lib.load().wdb_dueling_unfold_grads(
            _lib.stream_ptr(), ctypes.byref(self.online.struct())), "dueling_unfold_grads")
        return self.sums


NOISY_UPDATE, NOISY_ACTING = 0, 1            # the noise counter's domains (include/wdb200.h)


class NoisyHead:
    """A noisy network's head layers (FullyConnectedQ.noisy_layers()) as the struct
    wdb_noisy_net, with their effective layers in buffers of their own and, with grads, scratch
    for the effective layers' gradients."""

    def __init__(self, model, grads=False):
        self.model = model
        self.noisy = model.noisy_layers()
        dev = next(model.parameters()).device

        def buffers():
            return [(torch.zeros(L.out_features, L.in_features, device=dev),
                     torch.zeros(L.out_features, device=dev)) for L in self.noisy]
        self.layers = buffers()                  # [(W, b)], one per noisy layer
        self.grads = buffers() if grads else None
        self._index = {id(L): i for i, L in enumerate(self.noisy)}

    @staticmethod
    def shape(model):
        n = _lib.NoisyNet()
        layers = model.noisy_layers()
        n.n_layers = len(layers)
        if len(layers) > _lib.NOISY_MAX_LAYERS:
            return None
        for s, L in zip(n.layer, layers):
            s.in_dim, s.out_dim = int(L.in_features), int(L.out_features)
        return n

    def _pointers(self):
        tensors = [t for L in self.noisy for t in (L.weight_mu, L.weight_sigma, L.bias_mu,
                                                    L.bias_sigma, L.noise_in, L.noise_out)]
        tensors += [t for pair in self.layers + (self.grads or []) for t in pair]
        if self.grads is not None:
            tensors += [p.grad for L in self.noisy for p in (L.weight_mu, L.weight_sigma,
                                                             L.bias_mu, L.bias_sigma)]
        return tuple(None if t is None else t.data_ptr() for t in tensors)

    def struct(self):
        """The struct, rebuilt only when a tensor it points to has moved (load_state_dict keeps
        storage; .to() does not)."""
        key = self._pointers()
        if getattr(self, "_cached", None) is None or self._cached[0] != key:
            self._cached = (key, self._build())
        return self._cached[1]

    def _build(self):
        n = self.shape(self.model)
        for i, (s, L) in enumerate(zip(n.layer, self.noisy)):
            s.weight_mu, s.weight_sigma = _lib.ptr(L.weight_mu.data), _lib.ptr(L.weight_sigma.data)
            s.bias_mu, s.bias_sigma = _lib.ptr(L.bias_mu.data), _lib.ptr(L.bias_sigma.data)
            s.noise_in, s.noise_out = _lib.ptr(L.noise_in), _lib.ptr(L.noise_out)
            s.weight, s.bias = _lib.ptr(self.layers[i][0]), _lib.ptr(self.layers[i][1])
            if self.grads is not None:
                s.grad_weight, s.grad_bias = _lib.ptr(self.grads[i][0]), _lib.ptr(self.grads[i][1])
                s.grad_weight_mu = _lib.ptr(L.weight_mu.grad)
                s.grad_weight_sigma = _lib.ptr(L.weight_sigma.grad)
                s.grad_bias_mu, s.grad_bias_sigma = (_lib.ptr(L.bias_mu.grad),
                                                     _lib.ptr(L.bias_sigma.grad))
        return n

    def source(self, layer):
        """A DuelingFold source: the effective layer (and gradient scratch) of a noisy stream
        layer."""
        i = self._index[id(layer)]
        w, b = self.layers[i]
        gw, gb = self.grads[i] if self.grads is not None else (None, None)
        return w, b, gw, gb


def draw_noise(model, seed, domain, count, row0=0, rows=None):
    """wdb_noisy_draw into `rows` ([(noise_in [R, in], noise_out [R, out])] per noisy layer,
    counter rows row0 .. row0 + R - 1) or, by default, into the layers' own buffers (R = 1):
    one launch."""
    layers = model.noisy_layers()
    rows = rows if rows is not None else [(L.noise_in, L.noise_out) for L in layers]
    n = NoisyHead.shape(model)
    for s, (fi, fo) in zip(n.layer, rows):
        s.noise_in, s.noise_out = _lib.ptr(fi), _lib.ptr(fo)
    n_rows = rows[0][0].numel() // layers[0].in_features
    _lib.check(_lib.load().wdb_noisy_draw(_lib.stream_ptr(), ctypes.byref(n), int(seed),
                                          int(domain), int(count), int(row0), int(n_rows)),
               "noisy_draw")


def materialize(online, target, seed, update):
    """wdb_noisy_materialize of two NoisyHeads (online: row 0, target: row 1): one launch."""
    t = None if target is None else ctypes.byref(target.struct())
    _lib.check(_lib.load().wdb_noisy_materialize(
        _lib.stream_ptr(), ctypes.byref(online.struct()), t, int(seed), int(update)),
        "noisy_materialize")


def noisy_grads(head):
    """wdb_noisy_grads of a NoisyHead with grads: one launch."""
    _lib.check(_lib.load().wdb_noisy_grads(_lib.stream_ptr(), ctypes.byref(head.struct())),
               "noisy_grads")


class FusedNoisyUpdate:
    """One update of a noisy DQN or C51 policy, plain or dueling: wdb_noisy_materialize of the
    online and the target head under update `update`'s noise (1 launch), for a dueling head
    wdb_dueling_fold of the materialized streams (1 launch), the plain pass -- FusedDQNUpdate or
    FusedC51Update -- on the live trunk layers and the materialized (folded) head (2 launches),
    wdb_dueling_unfold_grads into the streams' gradient scratch (1 launch, dueling), then
    wdb_noisy_grads onto mu and sigma (1 launch).  Sums and outputs are the plain pass's."""

    plain_type = staticmethod(FusedDuelingUpdate.plain_type)

    @classmethod
    def supported(cls, algo, q_net, n_envs, n_agents, capacity, replay_rows):
        """True if a noisy FullyConnectedQ or FullyConnectedCategoricalQ's materialized network
        (folded, for a dueling head) is in the plain pass's envelope."""
        if type(q_net) not in (FullyConnectedQ, FullyConnectedCategoricalQ) or not q_net.noisy:
            return False
        if not (_masked(q_net) or isinstance(q_net.observation_space, Box)):
            return False
        shape = NoisyHead.shape(q_net)
        if shape is None or not _lib.load().wdb_noisy_supported(ctypes.byref(shape)):
            return False
        if q_net.dueling:
            if len(folded_widths(q_net)) > 3:
                return False
            if not _lib.load().wdb_dueling_fold_supported(
                    ctypes.byref(dueling_shape(q_net.policy_head))):
                return False
            u = _dueling_shape_struct(algo, q_net, n_envs, n_agents, capacity)
        else:
            if len(q_net.fc_dims) > 3:
                return False
            u = _shape_struct(algo, q_net, n_envs, n_agents, capacity)
        return cls.plain_type(q_net).fits(u, q_net, replay_rows)

    def __init__(self, algo, q_net, target_net, n_envs, n_agents, capacity, replay_rows, seed):
        self.seed = int(seed)
        self.online, self.target = NoisyHead(q_net, grads=True), NoisyHead(target_net)
        self.dueling = q_net.dueling
        if self.dueling:
            self.fold_online = DuelingFold(q_net, grads=True, source=self.online.source)
            self.fold_target = DuelingFold(target_net, source=self.target.source)
            u = _dueling_shape_struct(algo, q_net, n_envs, n_agents, capacity)
        else:
            u = _shape_struct(algo, q_net, n_envs, n_agents, capacity)
        self.plain = self.plain_type(q_net)(
            algo, q_net, target_net, n_envs, n_agents, capacity, replay_rows, u=u,
            point=self._point)
        self.rows, self.sums = self.plain.rows, self.plain.sums

    def _point(self, u):
        pairs = ((u.q, self.online, getattr(self, "fold_online", None), True),
                 (u.target_q, self.target, getattr(self, "fold_target", None), False))
        for net, noisy, folded, grads in pairs:
            fc = noisy.model.fc
            trunk = [(fc[str(i)][0].weight, fc[str(i)][0].bias) for i in range(len(fc))]
            head = folded.layers if folded is not None else noisy.layers
            for i, (w, b) in enumerate(trunk + head):
                net.w[i], net.b[i] = _lib.ptr(w.data), _lib.ptr(b.data)
            if grads:
                head = folded.grads if folded is not None else noisy.grads
                for i, (w, b) in enumerate([(w.grad, b.grad) for w, b in trunk] + head):
                    net.gw[i], net.gb[i] = _lib.ptr(w), _lib.ptr(b)

    def launch(self, obs, actions, rewards, done, windows, outputs=None, weights=None, update=0,
               action_mask=None):
        """The network's gradient (trunk, mu and sigma) into its `.grad` under update `update`'s
        noise; the other arguments are FusedQUpdate.launch's, and a masked network's
        `action_mask` for its masked pass."""
        materialize(self.online, self.target, self.seed, update)
        if self.dueling:
            fold(self.fold_online, self.fold_target)
        self.plain.launch(obs, actions, rewards, done, windows, outputs, weights,
                          **_mask_kwargs(action_mask))
        if self.dueling:
            _lib.check(_lib.load().wdb_dueling_unfold_grads(
                _lib.stream_ptr(), ctypes.byref(self.fold_online.struct())),
                "dueling_unfold_grads")
        noisy_grads(self.online)
        return self.sums


# The envelope checks by their function names: each is the class's `supported`.
fused_dqn_supported = FusedDQNUpdate.supported
fused_qr_dqn_supported = FusedQRDQNUpdate.supported
fused_iqn_supported = FusedIQNUpdate.supported
fused_c51_supported = FusedC51Update.supported
fused_dueling_supported = FusedDuelingUpdate.supported
fused_noisy_supported = FusedNoisyUpdate.supported
fused_branching_dqn_supported = FusedBranchingDQNUpdate.supported
