"""Float64 NumPy restatement of one discrete-action SAC update over sampled windows
(wdb_sac_discrete_{critic,actor}_update_sampled, include/wdb200.h; algorithms/sac_discrete.py):
the log-softmax policy, the exact soft value V' at obs', DQN's n-step return, both critics'
mse gradients, the actor's gradient through the twin minimum, log_alpha's gradient and the
passes' sums."""
import numpy as np

from dqn_update_reference import forward, gather


def log_softmax(z):
    m = z.max(axis=1, keepdims=True)
    s = z - m
    return s - np.log(np.exp(s).sum(axis=1, keepdims=True))


def backward(L, inputs, d):
    """[dW, db per layer] of the head delta d [B, out] through the MLP L (ReLU hidden layers)
    whose layer inputs are `inputs`."""
    grads = [None] * len(L)
    for i in reversed(range(len(L))):
        w, _ = L[i]
        grads[i] = (d.T @ inputs[i], d.sum(axis=0))
        if i > 0:
            d = (d @ w) * (inputs[i] > 0)
    return [g for pair in grads for g in pair]


def critic_pass(La, Lq1, Lq2, Lt1, Lt2, ring, windows, n_step, gamma, alpha):
    """{"grads1", "grads2", "q1", "q2", "returns", "boot", "sum_e1", "sum_e2"} of the critic
    pass; La / Lq1 / ... are [(W, b)] of the actor, the critics and the target critics."""
    Np = ring[0].shape[2]
    obs, actions, rewards, done, boot_obs = gather(ring, windows, n_step, Np)
    B = obs.shape[0]
    log_pi = log_softmax(forward(La, boot_obs)[0])
    m = np.minimum(forward(Lt1, boot_obs)[0], forward(Lt2, boot_obs)[0])
    boot = (np.exp(log_pi) * (m - alpha * log_pi)).sum(axis=1)
    R = boot
    for j in reversed(range(n_step)):
        R = np.where(done[j] != 0, 0.0, 1.0) * gamma * R + rewards[j]
    out = {"returns": R, "boot": boot}
    for k, L in (("1", Lq1), ("2", Lq2)):
        qs, inputs = forward(L, obs)
        q = qs[np.arange(B), actions]
        d = np.zeros_like(qs)
        d[np.arange(B), actions] = 2.0 * (q - R) / B
        out["grads" + k] = backward(L, inputs, d)
        out["q" + k] = q
        out["sum_e" + k] = float(((q - R) ** 2).sum())
    return out


def actor_pass(La, Lq1, Lq2, ring, windows, n_step, alpha, target_entropy):
    """{"grads", "entropies", "sum_m", "sum_log_pi", "loss", "alpha_grad"} of the actor pass:
    the gradient of (1/B) sum_g sum_a pi_a (alpha log pi_a - min(Q1, Q2)_a)."""
    Np = ring[0].shape[2]
    obs = gather(ring, windows, n_step, Np)[0]
    B = obs.shape[0]
    z, inputs = forward(La, obs)
    log_pi = log_softmax(z)
    pi = np.exp(log_pi)
    m = np.minimum(forward(Lq1, obs)[0], forward(Lq2, obs)[0])
    h = alpha * log_pi - m
    d = pi * (h - (pi * h).sum(axis=1, keepdims=True)) / B
    sum_log_pi = float((pi * log_pi).sum())
    return {"grads": backward(La, inputs, d), "entropies": -(pi * log_pi).sum(axis=1),
            "sum_m": float((pi * m).sum()), "sum_log_pi": sum_log_pi,
            "loss": float((pi * h).sum() / B), "alpha_grad": -(sum_log_pi / B + target_entropy)}
