"""Running reward scaling for A2C / PPO (policy keys `scale_rewards` and `reward_clip`): the
return half of SB3's `VecNormalize`.

Each (env, agent) row carries its running discounted return under the policy's own `gamma`.
After a rollout and before the update, one scan extends the carried returns through the batch
(restarting them where an episode ended), the batch's returns are merged into the policy's
running statistics of the return, and the update trains on clamp(r / sqrt(var + 1e-8), ±clip)
under the updated statistics; the mean is not subtracted.  The batch arrays keep the raw
rewards.

The statistics are buffers of the policy's model, so checkpoints carry them: float64
`return_count`, `return_mean` [1], `return_m2` [1] and the float32 `return_shift` [1] (the
mean) and `return_scale` [1] (count 0: 0 and 1), updated in place.  The per-row carry belongs to
the trainer and restarts at 0 whenever the trainer restarts the envs.  Native code:
csrc/wdb_reward_scale.cu (the scan), then wdb_obs_moments_* and wdb_obs_normalize with F = 1.
"""
import ctypes
import math

import torch

from warp_drive_b200 import lib as _lib
from warp_drive_b200.training import obs_norm

DEFAULT_CLIP = 10.0
_KEYS = ("scale_rewards", "reward_clip")


def reward_scale_settings(policy_config, policy):
    """(enabled, clip) of a policy config, validated; `policy` names it in the messages."""
    on = policy_config.get("scale_rewards", False)
    if not isinstance(on, bool):
        raise ValueError(f"policy '{policy}': scale_rewards is true or false, got {on!r}")
    if "reward_clip" not in policy_config:
        return on, DEFAULT_CLIP
    clip = policy_config["reward_clip"]
    if not on:
        raise ValueError(f"policy '{policy}': reward_clip needs scale_rewards: true, got "
                         f"reward_clip {clip!r} without it")
    if (isinstance(clip, bool) or not isinstance(clip, (int, float)) or not math.isfinite(clip)
            or clip <= 0):
        raise ValueError(f"policy '{policy}': reward_clip is a finite number > 0, got {clip!r}")
    return on, float(clip)


def refuse_reward_scale(config, trainer_name):
    """The replay trainers store raw rewards and sample them many iterations later: scaling
    them when sampled is a design of its own.  Refuse the keys there."""
    for policy, policy_config in config.get("policy", {}).items():
        for k in _KEYS:
            if policy_config.get(k) not in (None, False):
                raise ValueError(f"{trainer_name} does not take {k} (policy '{policy}'): reward "
                                 "scaling is for A2C / PPO (Trainer)")


def register_buffers(model):
    """The statistics of the return: no samples, so the identity."""
    model.register_buffer("return_count", torch.zeros((), dtype=torch.float64))
    model.register_buffer("return_mean", torch.zeros(1, dtype=torch.float64))
    model.register_buffer("return_m2", torch.zeros(1, dtype=torch.float64))
    model.register_buffer("return_shift", torch.zeros(1, dtype=torch.float32))
    model.register_buffer("return_scale", torch.ones(1, dtype=torch.float32))


class RewardScaler:
    """One trained policy's reward scaling: the per-row carry [E, Np], the batch's returns and
    the scaled rewards [T, E, Np] the update reads, all allocated once."""

    def __init__(self, model, shape, gamma, clip, device):
        T, E, Np = shape
        self.model, self.clip = model, float(clip)
        self.gamma = ctypes.c_float(gamma)           # the policy's gamma rounded to float32
        self.carry = torch.zeros((E, Np), dtype=torch.float32, device=device)
        self.returns = torch.empty((T, E, Np), dtype=torch.float32, device=device)
        self.scaled = torch.empty((T, E, Np), dtype=torch.float32, device=device)
        self._zero_shift = torch.zeros(1, dtype=torch.float32, device=device)

    def reset(self):
        """The envs restarted: every row's running return starts again at 0."""
        self.carry.zero_()

    def scale(self, rewards, done, num_devices=1):
        """The scan, the statistics update and the scaling of the raw batch rewards [T, E, Np]
        under done [T, E] (int32): four launches (plus one all-gather on several GPUs), no host
        wait.  Returns the scaled batch."""
        if (rewards.shape != self.scaled.shape or rewards.dtype != torch.float32
                or not rewards.is_contiguous() or done.dtype != torch.int32
                or tuple(done.shape) != tuple(rewards.shape[:2]) or not done.is_contiguous()):
            raise ValueError(f"scale_rewards: rewards f32 {tuple(self.scaled.shape)} and done "
                             f"i32 {tuple(self.scaled.shape[:2])} contiguous, got "
                             f"{rewards.dtype} {tuple(rewards.shape)}, {done.dtype} "
                             f"{tuple(done.shape)}")
        T, E, Np = rewards.shape
        L, s = _lib.load(), _lib.stream_ptr()
        _lib.check(L.wdb_discounted_return_scan(
            s, _lib.ptr(rewards), _lib.ptr(done), T, E, Np, self.gamma, _lib.ptr(self.carry),
            _lib.ptr(self.returns)), "discounted_return_scan")
        obs_norm.update_moments(self.model, self.returns.view(-1, 1), num_devices,
                                prefix="return")
        # (r - 0) * scale is exact in its subtract: clamp(r * scale, -clip, clip)
        _lib.check(L.wdb_obs_normalize(
            _lib.stream_ptr(), _lib.ptr(rewards), _lib.ptr(self.scaled), rewards.numel(), 1,
            _lib.ptr(self._zero_shift), _lib.ptr(self.model.return_scale),
            ctypes.c_float(self.clip)), "obs_normalize")
        return self.scaled
