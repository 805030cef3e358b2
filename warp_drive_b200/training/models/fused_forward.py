"""Rollout-time forward of a FullyConnected policy on the tensor cores:
`wdb_mlp_policy_forward` (csrc/wdb_mlp.cu, wgmma), one kernel per policy instead
of the 12-kernel torch module call.  The torch module stays the owner of the parameters
(training / autograd go through it); this wrapper re-packs them into the kernel's bf16
layout whenever they changed (`refresh()` after an optimizer step).
"""
import ctypes

import torch

from warp_drive_b200 import lib as _lib


class FusedPolicyForward:
    @staticmethod
    def supported(model):
        """Two hidden layers of equal width (multiple of 32, <= 256), one or two softmax heads;
        Box or Dict observations (a Dict's action mask goes to __call__ as `mask`)."""
        try:
            if getattr(model, "is_deterministic", True) or len(model.fc) != 2:
                return False
            # (a memoryless forward: it would drop a recurrent policy's state)
            if getattr(model, "is_recurrent", False):
                return False
            # (this forward reads raw observations)
            if getattr(model, "normalize_observations", False):
                return False
            dims = list(model.fc_dims)
            if dims[0] != dims[1] or len(model.output_dims) not in (1, 2):
                return False
            heads = [int(a) for a in model.output_dims] + [0]
            L = _lib.load()
            return L.wdb_mlp_blob_bytes(int(model.flattened_obs_size), int(dims[0]),
                                        heads[0], heads[1]) > 0
        except Exception:  # noqa: BLE001
            return False

    def __init__(self, model):
        assert self.supported(model)
        self.model = model
        self.F = int(model.flattened_obs_size)
        self.H = int(model.fc_dims[0])
        heads = [int(a) for a in model.output_dims] + [0]
        self.A0, self.A1 = heads[0], heads[1]          # A1 == 0: single-head policy
        self.lib = _lib.load()
        nbytes = int(self.lib.wdb_mlp_blob_bytes(self.F, self.H, self.A0, self.A1))
        dev = next(model.parameters()).device
        self.blob = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
        # whether this shape's forward can also sample both heads (wdb_mlp_policy_forward_sampled)
        self.samples = bool(self.lib.wdb_mlp_forward_samples(self.F, self.H, self.A0, self.A1))
        self.refresh()

    def refresh(self):
        """Re-pack the module's current parameters (call after every optimizer step)."""
        m = self.model
        l1, l2 = m.fc["0"][0], m.fc["1"][0]
        h0 = m.policy_head[0]
        h1 = m.policy_head[1] if self.A1 > 0 else None
        ts = [l1.weight, l1.bias, l2.weight, l2.bias, h0.weight, h0.bias,
              h1.weight if h1 is not None else None, h1.bias if h1 is not None else None,
              m.vf_head.weight, m.vf_head.bias]
        ts = [t.detach().float().contiguous() if t is not None else None for t in ts]
        _lib.check(self.lib.wdb_mlp_pack_weights(
            _lib.stream_ptr(), _lib.ptr(self.blob), *[_lib.ptr(t) for t in ts],
            self.F, self.H, self.A0, self.A1), "mlp_pack_weights")
        self._keep = ts

    def sampling(self, actions, agent_of_slot, n_agents, rng_state=None, uniforms=None,
                 env_begin=0):
        """The sampling arguments of a forward (see `__call__`): both heads' actions of every
        row go to `actions` [E, Np, 2] int32; row env * Np + slot is agent
        env * n_agents + agent_of_slot[slot] of the RNG state (or of `uniforms` [E, N, 2]).
        env_begin: the forward's rows are those of envs env_begin, env_begin + 1, ... (its
        obs, probabilities and `actions` start at env env_begin's rows)."""
        s = _lib.MlpSampling()
        s.actions, s.rng_state, s.uniforms = _lib.ptr(actions), _lib.ptr(rng_state), _lib.ptr(uniforms)
        s.agent_of_slot = _lib.ptr(agent_of_slot)
        s.n_agents, s.n_policy_agents = int(n_agents), int(agent_of_slot.numel())
        s.row_offset = int(env_begin) * s.n_policy_agents
        return s

    def _sampled(self, input_, tiles, rows, probs0, probs1, values, sampling):
        _lib.check(self.lib.wdb_mlp_policy_forward_sampled(
            _lib.stream_ptr(), _lib.ptr(self.blob), self.F, self.H, self.A0, self.A1,
            _lib.ptr(input_), int(tiles), int(rows), _lib.ptr(probs0), _lib.ptr(probs1),
            _lib.ptr(values), ctypes.byref(sampling)), "mlp_policy_forward_sampled")

    def __call__(self, obs, probs0, probs1, values=None, max_ctas=0, mask=None, sampling=None):
        """obs [..., F] float32 contiguous -> probs0 [..., A0], probs1 [..., A1] (written).
        max_ctas > 0 restricts the launch to that many SMs (side-by-side forwards).
        mask [..., A0 + A1] float32 contiguous (1 = valid): the masked forward.
        sampling (from `sampling()`, shapes with `samples` only): also sample both heads."""
        rows = obs.numel() // self.F
        _lib.check(self.lib.wdb_set_option(b"mlp_max_ctas", int(max_ctas)), "set_option")
        if sampling is not None:
            assert mask is None
            self._sampled(obs, False, rows, probs0, probs1, values, sampling)
            return
        if mask is not None:
            assert mask.dtype == torch.float32 and mask.numel() == rows * (self.A0 + self.A1)
            _lib.check(self.lib.wdb_mlp_policy_forward_masked(
                _lib.stream_ptr(), _lib.ptr(self.blob), self.F, self.H, self.A0, self.A1,
                _lib.ptr(obs), rows, _lib.ptr(mask), _lib.ptr(probs0), _lib.ptr(probs1),
                _lib.ptr(values)), "mlp_policy_forward_masked")
            return
        _lib.check(self.lib.wdb_mlp_policy_forward(
            _lib.stream_ptr(), _lib.ptr(self.blob), self.F, self.H, self.A0, self.A1,
            _lib.ptr(obs), rows, _lib.ptr(probs0), _lib.ptr(probs1), _lib.ptr(values)),
            "mlp_policy_forward")

    # ---- bf16 A-operand tiles (the MMA-ready copy of the observations) ----------------
    def tiles_bytes(self, rows):
        return int(self.lib.wdb_mlp_obs_tiles_bytes(self.F, int(rows)))

    def pack_obs(self, obs, tiles):
        """fp32 obs [..., F] -> `tiles` (uint8 tensor of tiles_bytes(rows) bytes)."""
        rows = obs.numel() // self.F
        _lib.check(self.lib.wdb_mlp_pack_obs(_lib.stream_ptr(), _lib.ptr(obs), rows, self.F,
                                             _lib.ptr(tiles)), "mlp_pack_obs")

    def forward_tiles(self, tiles, rows, probs0, probs1, values=None, max_ctas=0, sampling=None):
        """The forward fed from the bf16 tiles (written by pack_obs or by the fused env step)."""
        _lib.check(self.lib.wdb_set_option(b"mlp_max_ctas", int(max_ctas)), "set_option")
        if sampling is not None:
            self._sampled(tiles, True, rows, probs0, probs1, values, sampling)
            return
        _lib.check(self.lib.wdb_mlp_policy_forward_tiles(
            _lib.stream_ptr(), _lib.ptr(self.blob), self.F, self.H, self.A0, self.A1,
            _lib.ptr(tiles), int(rows), _lib.ptr(probs0), _lib.ptr(probs1), _lib.ptr(values)),
            "mlp_policy_forward_tiles")



def forward_pair(fa, fb, obs_a, obs_b, probs_a, probs_b, ctas_b=0, weights_stable=False):
    """Both policies' forwards in ONE launch (wdb_mlp_policy_forward_pair): `fa` / `fb` are
    FusedPolicyForward objects, probs_* = [probs_head0, probs_head1].  weights_stable: neither
    weight blob was written by the kernel launched just before on this stream."""
    pair = _lib.MlpPair()
    for w, (f, obs, pr) in enumerate(((fa, obs_a, probs_a), (fb, obs_b, probs_b))):
        pair.blob[w] = _lib.ptr(f.blob)
        pair.F[w], pair.H[w], pair.A0[w], pair.A1[w] = f.F, f.H, f.A0, f.A1
        pair.obs[w] = _lib.ptr(obs)
        pair.rows[w] = obs.numel() // f.F
        pair.probs0[w] = _lib.ptr(pr[0])
        pair.probs1[w] = _lib.ptr(pr[1] if len(pr) > 1 else None)
        pair.values[w] = None
    pair.ctas_b = int(ctas_b)
    pair.flags = _lib.MLP_WEIGHTS_STABLE if weights_stable else 0
    _lib.check(fa.lib.wdb_mlp_policy_forward_pair(_lib.stream_ptr(), ctypes.byref(pair)),
               "mlp_policy_forward_pair")
