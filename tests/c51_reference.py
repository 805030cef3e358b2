"""Float64 NumPy restatement of one categorical DQN (C51) update over sampled windows
(wdb_c51_update_sampled, include/wdb200.h; algorithms/dqn.py CategoricalDQN): the online atom
logits at obs, the chooser's expectations and the target's distribution of a* at obs', the atom
targets by DQN's n-step recursion, clamped, Dopamine's dense projection onto the support, the
cross-entropy with optional importance weights, Q-bar, R-bar and every parameter gradient of the
online network."""
import numpy as np

from dqn_update_reference import forward, gather, returns
from test_ddpg_update_reference_cpu import layers


def make_c51_models(F, A, dims, N=51, v_min=-10.0, v_max=10.0, seed=0):
    """(online, target) FullyConnectedCategoricalQ in float64 on a stand-in env with Box(F)
    observations and Discrete(A) actions."""
    import torch

    from test_ddpg_update_reference_cpu import _Env
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.utils import spaces as sp

    env = _Env(F, 1)
    env.env.action_space = {0: sp.Discrete(A)}
    torch.manual_seed(seed)
    cfg = {"type": "fully_connected_categorical_q", "fc_dims": dims, "num_atoms": N,
           "v_min": v_min, "v_max": v_max}
    mk = lambda: ModelFactory.create("fully_connected_categorical_q")(  # noqa: E731
        env=env, model_config=cfg, policy="shared",
        policy_tag_to_agent_id_map={"shared": [0]}).double()
    return mk(), mk()


def softmax(x):
    e = np.exp(x - x.max(axis=-1, keepdims=True))
    return e / e.sum(axis=-1, keepdims=True)


def project(tz, p_boot, z, dz):
    """m_i = sum_j clip(1 - |Tz_j - z_i| / dz, 0, 1) p'_j: [B, N]."""
    pair = np.clip(1.0 - np.abs(tz[:, None, :] - z[None, :, None]) / dz, 0.0, 1.0)
    return (pair * p_boot[:, None, :]).sum(axis=2)


def c51_sampled(models, ring, windows, n_step, gamma, double_q, z, dz, weights=None):
    """{"grads": [dW, db per layer], "loss", "sum_loss", "sum_q", "qbar" [B], "rbar" [B],
    "m" [B, N], "tz" [B, N], "p_boot" [B, N], "best" [B], "chooser" [B, A] (the chooser's
    expectations at obs')}; z the support [N] and dz its spacing."""
    Lq, Lt = layers(models[0]), layers(models[1])
    z = np.asarray(z, dtype=np.float64)
    N = z.shape[0]
    Np = ring[0].shape[2]
    obs, actions, rewards, done, boot_obs = gather(ring, windows, n_step, Np)
    B = obs.shape[0]
    rows = np.arange(B)
    ls, inputs = forward(Lq, obs)
    A = ls.shape[1] // N
    lt = forward(Lt, boot_obs)[0].reshape(B, A, N)
    lc = forward(Lq, boot_obs)[0].reshape(B, A, N) if double_q else lt
    chooser = (softmax(lc) * z).sum(axis=2)
    best = np.argmax(chooser, axis=1)                               # the first maximum
    p_boot = softmax(lt[rows, best])
    tz = np.clip(returns(rewards[..., None], done[..., None], np.broadcast_to(z, (B, N)), gamma),
                 z[0], z[-1])
    m = project(tz, p_boot, z, dz)
    logit = ls.reshape(B, A, N)[rows, actions]
    p = softmax(logit)
    logp = logit - logit.max(axis=1, keepdims=True)
    logp = logp - np.log(np.exp(logp).sum(axis=1, keepdims=True))
    w = np.ones(B) if weights is None else np.asarray(weights, dtype=np.float64)
    row_loss = -(m * logp).sum(axis=1)
    dlogit = (w / B)[:, None] * (p * m.sum(axis=1, keepdims=True) - m)
    d = np.zeros_like(ls)
    for i in range(N):
        d[rows, actions * N + i] = dlogit[:, i]
    grads = [None] * len(Lq)
    for li in reversed(range(len(Lq))):
        W, _ = Lq[li]
        grads[li] = (d.T @ inputs[li], d.sum(axis=0))
        if li > 0:
            d = (d @ W) * (inputs[li] > 0)
    qbar, rbar = (p * z).sum(axis=1), (m * z).sum(axis=1)
    return {"grads": [g for pair in grads for g in pair], "loss": float((w * row_loss).mean()),
            "sum_loss": float((w * row_loss).sum()), "sum_q": float(qbar.sum()), "qbar": qbar,
            "rbar": rbar, "m": m, "tz": tz, "p_boot": p_boot, "best": best, "chooser": chooser}
