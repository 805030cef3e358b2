"""Float64 NumPy restatement of one TQC update over sampled windows
(wdb_tqc_{critic,actor}_update_sampled, include/wdb200.h; algorithms/tqc.py): SAC's squashed
sample at obs', the pooled target atoms of M critics truncated to the K smallest (a stable
sort), each kept atom's n-step return, the quantile Huber pair loss and each critic's gradient;
the actor's gradient through the mean of all quantiles, the tanh, the reparameterisation, the
clamp and the log-prob's own terms; log_alpha's gradient and the passes' sums.  Any M, N, d."""
import numpy as np

from ddpg_update_reference import _backward, _forward
from sac_update_reference import squashed


def make_ring(C, E, Np, F, A, seed=0):
    """obs [C, E, Np, F], actions [C, E, Np, A] in (-2, 2), rewards [C, E, Np], int32 done
    [C, E] in {0, 1}."""
    g = np.random.default_rng(seed)
    obs = g.standard_normal((C, E, Np, F))
    actions = g.uniform(-2.0, 2.0, (C, E, Np, A))
    rewards = g.standard_normal((C, E, Np))
    done = (g.random((C, E)) < 0.25).astype(np.int32)
    return obs, actions, rewards, done


def gather(ring, windows, n_step, Np):
    """obs [B, F], actions [B, A], rewards / done [n_step, B], bootstrap obs [B, F]."""
    obs, actions, rewards, done = ring
    C = obs.shape[0]
    s, n = windows[:, 0].astype(np.int64), windows[:, 1].astype(np.int64)
    steps = (s[None, :] + np.arange(n_step + 1)[:, None]) % C
    o = obs.reshape(C, -1, obs.shape[-1])
    a = actions.reshape(C, -1, actions.shape[-1])
    return (o[s, n], a[s, n], rewards.reshape(C, -1)[steps[:-1], n],
            done[steps[:-1], n // Np], o[steps[-1], n])


def quantile_fractions(N):
    """tau_i = (2i + 1) / (2N), rounded once to float32."""
    return ((2.0 * np.arange(N) + 1.0) / (2.0 * N)).astype(np.float32).astype(np.float64)


def _flat(grads):
    return [t for pair in grads for t in pair]


def critic_pass(La, Lcs, Lts, ring, windows, n_step, gamma, alpha, scale, bias, lo, hi, noise,
                n_drop):
    """The critic pass.  La: the actor's [(W, b)] (head 2A); Lcs, Lts: the M critics' and
    target critics' layers (head N); noise [B, A] (eps').  Returns {"grads" [M][dW, db, ...],
    "theta" [B, M, N], "returns" [B, K], "q_means", "target_means" [B], "loss", "sum_loss",
    "sum_q", "atoms" [B, M N]}."""
    Np = ring[0].shape[2]
    obs, actions, rewards, done, boot_obs = gather(ring, windows, n_step, Np)
    B, A = actions.shape
    M, N = len(Lcs), Lcs[0][-1][0].shape[0]
    K = M * (N - n_drop)
    s = squashed(_forward(La, boot_obs)[0][-1], noise, A, lo, hi)
    x_t = np.concatenate([boot_obs, scale * s["y"] + bias], axis=1)
    atoms = np.concatenate([_forward(L, x_t)[0][-1] for L in Lts], axis=1)
    kept = np.take_along_axis(atoms, np.argsort(atoms, axis=1, kind="stable")[:, :K], axis=1)
    T = kept - alpha * s["log_pi"][:, None]
    for j in reversed(range(n_step)):
        T = (1.0 - done[j])[:, None] * gamma * T + rewards[j][:, None]
    tau = quantile_fractions(N)[None, :, None]
    c = 1.0 / (B * M * N * K)
    x = np.concatenate([obs, actions], axis=1)
    grads, thetas, loss_rows = [], [], np.zeros(B)
    for L in Lcs:
        acts, masks, _ = _forward(L, x)
        theta = acts[-1]
        u = T[:, None, :] - theta[:, :, None]
        w = np.abs(tau - (u < 0))
        au = np.abs(u)
        loss_rows += (w * np.where(au <= 1.0, 0.5 * u * u, au - 0.5)).sum(axis=(1, 2))
        g, _ = _backward(L, acts, masks, -c * (w * np.clip(u, -1.0, 1.0)).sum(axis=2))
        grads.append(_flat(g))
        thetas.append(theta)
    theta = np.stack(thetas, axis=1)
    q_means = theta.mean(axis=(1, 2))
    return {"grads": grads, "theta": theta, "returns": T, "q_means": q_means,
            "target_means": T.mean(axis=1), "loss": float(loss_rows.sum() * c),
            "sum_loss": float(loss_rows.sum()), "sum_q": float(q_means.sum()), "atoms": atoms}


def actor_pass(La, Lcs, ring, windows, n_step, alpha, scale, bias, lo, hi, noise,
               target_entropy):
    """The actor pass with eps = noise [B, A]: {"grads" [dW, db, ...], "log_probs", "q_bar"
    [B], "sum_q", "sum_log_pi", "loss", "alpha_grad"}."""
    Np = ring[0].shape[2]
    obs = gather(ring, windows, n_step, Np)[0]
    B, F = obs.shape
    A = noise.shape[1]
    M, N = len(Lcs), Lcs[0][-1][0].shape[0]
    a_acts, ma, _ = _forward(La, obs)
    s = squashed(a_acts[-1], noise, A, lo, hi)
    x = np.concatenate([obs, scale * s["y"] + bias], axis=1)
    q_sum, da = np.zeros(B), np.zeros((B, A))
    for L in Lcs:
        acts, masks, _ = _forward(L, x)
        q_sum += acts[-1].sum(axis=1)
        _, dx = _backward(L, acts, masks, np.full((B, N), -1.0 / (B * M * N)), input_grad=True)
        da += dx[:, F:]
    q_bar = q_sum / (M * N)
    d_lp = alpha / B
    du = da * scale * (1.0 - s["y"] ** 2) + d_lp * 2.0 * s["y"]
    dls = np.where(s["in_range"], du * s["sig"] * noise - d_lp, 0.0)
    ga, _ = _backward(La, a_acts, ma, np.concatenate([du, dls], axis=1))
    sum_log_pi = float(s["log_pi"].sum())
    return {"grads": _flat(ga), "log_probs": s["log_pi"], "q_bar": q_bar,
            "sum_q": float(q_bar.sum()), "sum_log_pi": sum_log_pi,
            "loss": float((alpha * s["log_pi"] - q_bar).mean()),
            "alpha_grad": -(sum_log_pi / B + target_entropy)}
