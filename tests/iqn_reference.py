"""Float64 NumPy restatement of one implicit quantile network update over sampled windows
(wdb_iqn_update_sampled, include/wdb200.h; algorithms/dqn.py ImplicitQuantileDQN): both trunks
on obs and obs', the tau embeddings and c-bar over the K midpoints, the bootstrap action a*, the
N' targets by DQN's n-step recursion, the quantile Huber loss with optional importance weights,
Q-bar, R-bar and every parameter gradient of the online network -- trunk, head and embedding."""
import numpy as np

from dqn_update_reference import gather, returns


def make_iqn_models(F, A, dims, n_cos=8, N=4, NP=5, K=6, seed=0):
    """(online, target) FullyConnectedIQN in float64 on a stand-in env with Box(F) observations
    and Discrete(A) actions."""
    import torch

    from test_ddpg_update_reference_cpu import _Env
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.utils import spaces as sp

    env = _Env(F, 1)
    env.env.action_space = {0: sp.Discrete(A)}
    torch.manual_seed(seed)
    cfg = {"type": "fully_connected_iqn", "fc_dims": dims, "num_cosines": n_cos,
           "num_tau_samples": N, "num_tau_prime_samples": NP, "num_quantile_samples": K}
    mk = lambda: ModelFactory.create("fully_connected_iqn")(  # noqa: E731
        env=env, model_config=cfg, policy="shared",
        policy_tag_to_agent_id_map={"shared": [0]}).double()
    return mk(), mk()


def parts(model):
    """([(W, b)] of the trunk, (W, b) of the head, (E, e) of the embedding), as float64 NumPy
    (of a float32 model too: the reference computes in float64)."""
    np_ = lambda lin: (lin.weight.detach().double().cpu().numpy(),  # noqa: E731
                       lin.bias.detach().double().cpu().numpy())
    trunk = [np_(model.fc[str(i)][0]) for i in range(len(model.fc))]
    return trunk, np_(model.policy_head), np_(model.tau_embedding)


def trunk_forward(trunk, x):
    """psi(x) and the layer inputs (for the backward)."""
    inputs = []
    for w, b in trunk:
        inputs.append(x)
        x = np.maximum(x @ w.T + b, 0.0)
    return x, inputs


def cos_features(taus, n_cos):
    return np.cos(taus[..., None] * (np.pi * np.arange(n_cos)))


def embedding(emb, taus):
    """(phi(tau), the cosine features)."""
    cf = cos_features(taus, emb[0].shape[1])
    return np.maximum(cf @ emb[0].T + emb[1], 0.0), cf


def midpoints(K):
    return (2 * np.arange(K) + 1) / (2 * K)


def huber(u, kappa):
    au = np.abs(u)
    return np.where(au < kappa, 0.5 * u * u, kappa * (au - 0.5 * kappa))


def iqn_sampled(models, ring, windows, n_step, gamma, kappa, double_q, taus, weights=None):
    """{"grads": [dW, db per trunk layer, head, embedding], "loss", "sum_loss", "sum_q", "qbar"
    [B], "rbar" [B], "theta" [B, N], "targets" [B, N'], "u" [B, N, N'], "best" [B],
    "chooser" [B, A]} for taus [B, N + N']."""
    online, target = models
    N, K = online.num_tau_samples, online.num_quantile_samples
    (Tq, (Wh, bh), Eq), (Tt, (Wth, bth), Et) = parts(online), parts(target)
    Np = ring[0].shape[2]
    obs, actions, rewards, done, boot_obs = gather(ring, windows, n_step, Np)
    obs, rewards, boot_obs = (np.asarray(x, dtype=np.float64) for x in (obs, rewards, boot_obs))
    taus = np.asarray(taus, dtype=np.float64)
    B = obs.shape[0]
    rows = np.arange(B)
    tau, tau_p = taus[:, :N], taus[:, N:]
    psi, inputs = trunk_forward(Tq, obs)                             # [B, H]
    psi_t = trunk_forward(Tt, boot_obs)[0]
    # a*: the first argmax of the collapsed head, online (double_q) or target, at obs'
    if double_q:
        cbar = embedding(Eq, midpoints(K))[0].mean(axis=0)
        chooser = (trunk_forward(Tq, boot_obs)[0] * cbar) @ Wh.T + bh
    else:
        cbar = embedding(Et, midpoints(K))[0].mean(axis=0)
        chooser = (psi_t * cbar) @ Wth.T + bth
    best = np.argmax(chooser, axis=1)
    zt = (psi_t[:, None, :] * embedding(Et, tau_p)[0]) @ Wth.T + bth   # [B, N', A]
    T = returns(rewards[..., None], done[..., None], zt[rows, :, best], gamma)   # [B, N']
    NP = T.shape[1]
    phi, cf = embedding(Eq, tau)                                     # [B, N, H], [B, N, n_cos]
    mg = psi[:, None, :] * phi
    z = mg @ Wh.T + bh                                               # [B, N, A]
    theta = z[rows, :, actions]                                      # [B, N]
    u = T[:, None, :] - theta[:, :, None]                            # [B, i, j]
    m = np.abs(tau[:, :, None] - (u < 0))
    w = np.ones(B) if weights is None else np.asarray(weights, dtype=np.float64)
    row_loss = (m * huber(u, kappa) / kappa).sum(axis=(1, 2)) / NP
    dtheta = -(w / (B * NP * kappa))[:, None] * (m * np.clip(u, -kappa, kappa)).sum(axis=2)
    dz = np.zeros_like(z)
    dz[rows, :, actions] = dtheta
    head = (np.einsum("bia,bih->ah", dz, mg), dz.sum(axis=(0, 1)))
    dmg = dz @ Wh                                                    # [B, N, H]
    dpsi = (dmg * phi).sum(axis=1)
    dphi = dmg * psi[:, None, :] * (phi > 0)
    emb = (np.einsum("bih,bic->hc", dphi, cf), dphi.sum(axis=(0, 1)))
    d = dpsi * (psi > 0)
    grads = [None] * len(Tq)
    for li in reversed(range(len(Tq))):
        grads[li] = (d.T @ inputs[li], d.sum(axis=0))
        if li > 0:
            d = (d @ Tq[li][0]) * (inputs[li] > 0)
    qbar, rbar = theta.mean(axis=1), T.mean(axis=1)
    return {"grads": [g for pair in grads + [head, emb] for g in pair],
            "loss": float((w * row_loss).mean()), "sum_loss": float((w * row_loss).sum()),
            "sum_q": float(qbar.sum()), "qbar": qbar, "rbar": rbar, "theta": theta,
            "targets": T, "u": u, "best": best, "chooser": chooser}
