"""Float64 NumPy restatement of one branching DQN update over sampled windows
(wdb_branching_dqn_update_sampled / _prioritized, include/wdb200.h; algorithms/dqn.py
BranchingDQN), and the same pass with error bars for the native kernels.

Heads d = 0 .. D-1 have sizes A_d and offsets o_d = sum_{e<d} A_e; the network's head has
A = sum_d A_d columns and Q_d(s, .) is columns o_d .. o_d + A_d - 1.  Per window g with actions
a_d [B, D]:
  boot_d = target_d(obs')[first argmax online_d(obs')] (double_q) or max target_d(obs'),
  R      = DQN's n-step recursion on (1/D) sum_d boot_d,
  loss   = (1/B) sum_g w_g (1/D) sum_d huber(Q_d(obs, a_d) - R, delta),
  Q-bar  = (1/D) sum_d Q_d(obs, a_d)."""
import numpy as np

import q_update_bounds as qb
from dqn_update_reference import forward, gather, returns
from test_ddpg_update_reference_cpu import layers
from update_reference import D as DEPS
from update_reference import exact, f_div, f_mul, f_sub


def offsets(sizes):
    return np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)


def make_branching_models(F, sizes, dims, seed=0):
    """(online, target) FullyConnectedBranchingQ in float64 on a stand-in env with Box(F)
    observations and MultiDiscrete(sizes) actions (Discrete for one head)."""
    import torch

    from test_ddpg_update_reference_cpu import _Env
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.utils import spaces as sp

    env = _Env(F, 1)
    env.env.action_space = {0: (sp.Discrete(sizes[0]) if len(sizes) == 1
                                else sp.MultiDiscrete(list(sizes)))}
    torch.manual_seed(seed)
    cfg = {"type": "fully_connected_branching_q", "fc_dims": list(dims)}
    mk = lambda: ModelFactory.create("fully_connected_branching_q")(  # noqa: E731
        env=env, model_config=cfg, policy="shared",
        policy_tag_to_agent_id_map={"shared": [0]}).double()
    return mk(), mk()


def make_branching_ring(C, E, Np, F, sizes, seed=0):
    """obs [C, E, Np, F], int actions [C, E, Np, D], rewards [C, E, Np], done [C, E] in
    {0, 1, 2}."""
    g = np.random.default_rng(seed)
    obs = g.standard_normal((C, E, Np, F))
    actions = np.stack([g.integers(0, a, (C, E, Np)) for a in sizes], axis=-1).astype(np.int32)
    rewards = g.standard_normal((C, E, Np))
    done = g.choice(np.array([0, 1, 2], dtype=np.int32), size=(C, E), p=[0.7, 0.15, 0.15])
    return obs, actions, rewards, done


def gather_branching(ring, windows, n_step, Np):
    """dqn_update_reference.gather with the D actions of each window: actions [B, D]."""
    obs, actions, rewards, done = ring
    C, D = obs.shape[0], actions.shape[-1]
    o, _, r, d, ob = gather((obs, actions[..., 0:1], rewards, done), windows, n_step, Np)
    s, n = windows[:, 0].astype(np.int64), windows[:, 1].astype(np.int64)
    return o, actions.reshape(C, -1, D)[s, n], r, d, ob


def branching_sampled(models, ring, windows, n_step, gamma, delta, double_q, sizes,
                      weights=None):
    """{"grads": [dW, db per layer], "q" (Q-bar), "returns", "boot", "loss", "sum_huber",
    "sum_q"} of the pass in float64."""
    Lq, Lt = layers(models[0]), layers(models[1])
    Np = ring[0].shape[2]
    obs, actions, rewards, done, boot_obs = gather_branching(ring, windows, n_step, Np)
    B, Dh = actions.shape
    rows = np.arange(B)
    w = np.ones(B) if weights is None else np.asarray(weights, np.float64)
    qs, inputs = forward(Lq, obs)
    qt, _ = forward(Lt, boot_obs)
    chooser = forward(Lq, boot_obs)[0] if double_q else qt
    boot = np.zeros(B)
    for o, a in zip(offsets(sizes), sizes):
        best = o + np.argmax(chooser[:, o:o + a], axis=1)      # the first maximum
        boot += qt[rows, best]
    boot /= Dh
    R = returns(rewards, done, boot, gamma)
    cols = offsets(sizes)[None, :] + actions                     # [B, D]
    q = qs[rows[:, None], cols]
    diff = q - R[:, None]
    huber = np.where(np.abs(diff) < delta, 0.5 * diff * diff,
                     delta * (np.abs(diff) - 0.5 * delta))
    d = np.zeros_like(qs)
    for k in range(Dh):
        d[rows, cols[:, k]] += w * np.clip(diff[:, k], -delta, delta) / (B * Dh)
    grads = [None] * len(Lq)
    for i in reversed(range(len(Lq))):
        W, _ = Lq[i]
        grads[i] = (d.T @ inputs[i], d.sum(axis=0))
        if i > 0:
            d = (d @ W) * (inputs[i] > 0)
    row_loss = huber.mean(axis=1)
    return {"grads": [g for pair in grads for g in pair], "q": q.mean(axis=1), "returns": R,
            "boot": boot, "loss": float((w * row_loss).mean()),
            "sum_huber": float((w * row_loss).sum()), "sum_q": float(q.mean(axis=1).sum())}


def branching_pass(Lq, Lt, rows, gamma, kappa, double_q, sizes, weights=None):
    """The pass with error bars (tests/q_update_bounds.py's rules and helpers): rows are
    gather_branching's (obs, actions [B, D], rewards, done, boot_obs) in float32; Lq, Lt
    [(W, b)] float32 values in float64.  Returns qr_pass's dict: grads, q_values (Q-bar),
    returns, sums (2) and ok [B] (every premise of the row: the backward ReLU masks and, with
    double_q, each head's bootstrap argmax)."""
    obs, actions, rewards, done, boot_obs = rows
    obs, boot_obs = exact(np.asarray(obs, np.float64)), exact(np.asarray(boot_obs, np.float64))
    rewards = np.asarray(rewards, np.float64)
    actions = np.asarray(actions).astype(np.int64)
    kappa = qb.f32(kappa)
    B, Dh = actions.shape
    r = np.arange(B)
    qs, inputs, ok = qb.forward(Lq, obs, True)
    qt = qb.forward(Lt, boot_obs, False)[0]
    chooser = qb.forward(Lq, boot_obs, False)[0] if double_q else qt
    w = None if weights is None else exact(np.asarray(weights, np.float32).astype(np.float64))
    wv = np.ones(B) if weights is None else w[0]
    boots = []
    for o, a in zip(offsets(sizes), sizes):
        head = (chooser[0][:, o:o + a], chooser[1][:, o:o + a])
        if double_q:
            best, k = qb.first_argmax(head)
            ok &= k
            boots.append((qt[0][r, o + best], qt[1][r, o + best]))
        else:
            boots.append(qb.f_max((qt[0][:, o:o + a], qt[1][:, o:o + a])))
    total = qb.f_sum((np.stack([b[0] for b in boots], 1), np.stack([b[1] for b in boots], 1)))
    T = qb.nstep(f_div(total, exact(np.full(B, float(Dh)))), rewards, done, gamma)
    cols = offsets(sizes)[None, :] + actions
    q = (qs[0][r[:, None], cols], qs[1][r[:, None], cols])               # [B, D]
    diff = f_sub(q, (T[0][:, None], T[1][:, None]))
    c = qb.f_clip(diff, -kappa, kappa)
    if w is not None:
        c = f_mul(c, (w[0][:, None], w[1][:, None]))
    dq = f_mul(c, qb.norm_of(float(B) * Dh))
    dh = (np.zeros_like(qs[0]), np.zeros_like(qs[0]))
    for k in range(Dh):                     # one column per head: no two heads share a column
        dh[0][r, cols[:, k]], dh[1][r, cols[:, k]] = dq[0][:, k], dq[1][:, k]
    h, hb = qb.huber_terms(diff, kappa)
    scale = (wv / Dh)[:, None]
    t = (h * scale, hb * scale + (Dh + 4) * DEPS * h * scale)
    qbar = f_div(qb.f_sum(q), exact(np.full(B, float(Dh))))
    sums = [qb.double_sum(t, 16), qb.double_sum(qbar, 16)]
    grads = qb.backward(Lq, inputs, dh, qb.tile_depth(B))
    return {"grads": grads, "q_values": qbar, "returns": T, "sums": sums, "ok": ok}
