"""Float64 NumPy restatement of one quantile-regression DQN update over sampled windows
(wdb_qr_dqn_update_sampled, include/wdb200.h; algorithms/dqn.py QuantileDQN): the online
quantiles at obs, the target's and (double_q) the online network's at obs', the bootstrap action
a* (first argmax of the mean quantile), the N targets by DQN's n-step recursion, the quantile
Huber loss with optional importance weights, Q-bar, R-bar and every parameter gradient of the
online network."""
import numpy as np

from dqn_update_reference import forward, gather, returns
from test_ddpg_update_reference_cpu import layers


def make_qr_models(F, A, N, dims, seed=0):
    """(online, target) FullyConnectedQuantileQ with N quantiles in float64 on a stand-in env
    with Box(F) observations and Discrete(A) actions."""
    import torch

    from test_ddpg_update_reference_cpu import _Env
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.utils import spaces as sp

    env = _Env(F, 1)
    env.env.action_space = {0: sp.Discrete(A)}
    torch.manual_seed(seed)
    cfg = {"type": "fully_connected_quantile_q", "fc_dims": dims, "num_quantiles": N}
    mk = lambda: ModelFactory.create("fully_connected_quantile_q")(  # noqa: E731
        env=env, model_config=cfg, policy="shared",
        policy_tag_to_agent_id_map={"shared": [0]}).double()
    return mk(), mk()


def huber(u, kappa):
    au = np.abs(u)
    return np.where(au < kappa, 0.5 * u * u, kappa * (au - 0.5 * kappa))


def qr_dqn_sampled(models, ring, windows, n_step, gamma, kappa, double_q, N, weights=None):
    """{"grads": [dW, db per layer], "loss", "sum_loss", "sum_q", "qbar" [B], "rbar" [B],
    "theta" [B, N], "targets" [B, N], "u" [B, N, N], "best" [B]}."""
    Lq, Lt = layers(models[0]), layers(models[1])
    Np = ring[0].shape[2]
    obs, actions, rewards, done, boot_obs = gather(ring, windows, n_step, Np)
    B = obs.shape[0]
    rows = np.arange(B)
    qs, inputs = forward(Lq, obs)
    A = qs.shape[1] // N
    qt = forward(Lt, boot_obs)[0].reshape(B, A, N)
    chooser = forward(Lq, boot_obs)[0].reshape(B, A, N) if double_q else qt
    best = np.argmax(chooser.mean(axis=2), axis=1)                  # the first maximum
    T = returns(rewards[..., None], done[..., None], qt[rows, best], gamma)   # [B, N]
    theta = qs.reshape(B, A, N)[rows, actions]                       # [B, N]
    tau = (2 * np.arange(N) + 1) / (2 * N)
    u = T[:, None, :] - theta[:, :, None]                            # [B, i, j]
    m = np.abs(tau[None, :, None] - (u < 0))
    w = np.ones(B) if weights is None else np.asarray(weights, dtype=np.float64)
    row_loss = (m * huber(u, kappa) / kappa).sum(axis=(1, 2)) / N
    dtheta = -(w / (B * N * kappa))[:, None] * (m * np.clip(u, -kappa, kappa)).sum(axis=2)
    d = np.zeros_like(qs)
    for i in range(N):
        d[rows, actions * N + i] = dtheta[:, i]
    grads = [None] * len(Lq)
    for li in reversed(range(len(Lq))):
        W, _ = Lq[li]
        grads[li] = (d.T @ inputs[li], d.sum(axis=0))
        if li > 0:
            d = (d @ W) * (inputs[li] > 0)
    qbar, rbar = theta.mean(axis=1), T.mean(axis=1)
    return {"grads": [g for pair in grads for g in pair], "loss": float((w * row_loss).mean()),
            "sum_loss": float((w * row_loss).sum()), "sum_q": float(qbar.sum()), "qbar": qbar,
            "rbar": rbar, "theta": theta, "targets": T, "u": u, "best": best,
            "chooser": chooser}
