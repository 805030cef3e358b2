"""NumPy restatement of running reward scaling (training/reward_scale.py,
csrc/wdb_reward_scale.cu).

The scan is float32 in the kernel's order: ret = (gamma * carry) + r, each operation rounded on
its own (no FMA), then returns[t] = ret, then the carry restarts at 0 where done[t, env] > 0.
The statistics of the returns are obs_norm_reference's float64 moments with F = 1, and the
scaling its float32 normalization with a zero shift: clamp(r * scale, -clip, clip).
"""
import numpy as np

from obs_norm_reference import batch_moments, chan, normalize_f32, shift_scale


def scan_f32(rewards, done, gamma, carry):
    """(returns [T, E, Np], carry out [E, Np]) of rewards [T, E, Np] and done [T, E] from the
    incoming carry [E, Np], float32 with gamma rounded to float32."""
    r = np.asarray(rewards, dtype=np.float32)
    d = np.asarray(done)
    g = np.float32(gamma)
    c = np.array(carry, dtype=np.float32, copy=True)
    out = np.empty_like(r)
    for t in range(r.shape[0]):
        ret = np.add(np.multiply(g, c, dtype=np.float32), r[t], dtype=np.float32)
        out[t] = ret
        c = np.where((d[t] > 0)[:, None], np.float32(0.0), ret).astype(np.float32)
    return out, c


def scale_f32(rewards, scale, clip):
    """clamp(r * scale, -clip, clip) as wdb_obs_normalize with F = 1 and a zero shift."""
    r = np.asarray(rewards, dtype=np.float32)
    return normalize_f32(r.reshape(-1, 1), np.zeros(1, np.float32),
                         np.asarray(scale, np.float32).reshape(1), clip).reshape(r.shape)


class RunningReturns:
    """One policy's reward scaling on the host: the carry and the float64 statistics."""

    def __init__(self, E, Np, gamma, clip):
        self.gamma, self.clip = gamma, clip
        self.carry = np.zeros((E, Np), np.float32)
        self.stats = (0.0, np.zeros(1), np.zeros(1))

    def reset(self):
        self.carry[:] = 0

    def step(self, rewards, done):
        """Scan, then merge the returns into the statistics; returns the batch's returns."""
        returns, self.carry = scan_f32(rewards, done, self.gamma, self.carry)
        self.stats = chan(self.stats, batch_moments(returns.reshape(-1, 1)))
        return returns

    def scale(self):
        return shift_scale(*self.stats)[1]
