"""One policy's prioritized-replay store (Schaul et al. 2016, proportional): the leaves, sum tree,
running maximum priority and beta scalar of wdb_per_* (include/wdb200.h, csrc/wdb_per.cu) on
the device, and the buffers of one update's sample (priorities, importance-sampling weights)
and of the priorities' inputs (Q(obs, a), R).  Per GPU; not checkpointed."""
import ctypes

import torch

from warp_drive_b200 import lib as _lib


class PrioritizedReplay:
    def __init__(self, capacity, n_rows, n_step, rows, alpha, epsilon, device):
        """A store over `capacity` slots x `n_rows` agent rows of a ring with horizon n_step,
        sampled `rows` windows at a time."""
        self.lib = _lib.load()
        n_leaves = int(capacity) * int(n_rows)
        n_nodes = int(self.lib.wdb_per_nodes(n_leaves))
        if n_nodes < 0:
            raise ValueError(f"prioritized replay takes fewer than 2^31 windows, got {n_leaves}")
        self.levels = int(self.lib.wdb_per_levels(n_leaves))
        self.leaves = torch.zeros(n_leaves, dtype=torch.float32, device=device)
        self.nodes = torch.zeros(n_nodes, dtype=torch.float64, device=device)
        self.p_max = torch.ones(1, dtype=torch.float32, device=device)
        self.beta = torch.zeros(1, dtype=torch.float32, device=device)
        self._beta_value = None
        self.priorities, self.weights, self.q_values, self.returns = (
            torch.zeros(rows, dtype=torch.float32, device=device) for _ in range(4))
        s = self.store = _lib.PerStore()
        s.capacity, s.n_rows, s.n_step = int(capacity), int(n_rows), int(n_step)
        s.alpha, s.epsilon = float(alpha), float(epsilon)
        s.leaves, s.nodes, s.p_max = (_lib.ptr(t) for t in (self.leaves, self.nodes, self.p_max))

    def nbytes(self):
        """Device bytes of the store and its per-update buffers."""
        ts = (self.leaves, self.nodes, self.p_max, self.beta, self.priorities, self.weights,
              self.q_values, self.returns)
        return sum(t.numel() * t.element_size() for t in ts)

    def admit(self, before, after):
        """After a rollout: before / after are the ring's (cursor, filled)."""
        _lib.check(self.lib.wdb_per_admit(_lib.stream_ptr(), ctypes.byref(self.store),
                                          *before, *after), "per_admit")

    def set_beta(self, value):
        """The device beta the next samples' weights use (a fill only when it changes)."""
        if value != self._beta_value:
            self.beta.fill_(float(value))
            self._beta_value = value

    def sample(self, windows, seed, counter):
        """windows (int32 [rows, 2]) <- stratified proportional draws; fills priorities and
        weights."""
        _lib.check(self.lib.wdb_per_sample_windows(
            _lib.stream_ptr(), ctypes.byref(self.store), _lib.ptr(windows),
            _lib.ptr(self.priorities), _lib.ptr(self.weights), int(windows.shape[0]), seed,
            counter, _lib.ptr(self.beta)), "per_sample_windows")

    def set_priorities(self, windows, q_values, returns, oldest, filled):
        """The windows' leaves <- (|Q - R| + epsilon)^alpha (float32 [rows] each)."""
        _lib.check(self.lib.wdb_per_set_priorities(
            _lib.stream_ptr(), ctypes.byref(self.store), _lib.ptr(windows),
            int(windows.shape[0]), _lib.ptr(q_values), _lib.ptr(returns), int(oldest),
            int(filled)), "per_set_priorities")
