"""Float64 NumPy restatement of one DDPG update of one policy -- what `wdb_ddpg_update`
computes (include/wdb200.h) and what TrainerDDPG's torch update computes by autograd: five MLP
forwards, the n-step returns (DDPG.n_step_returns), both losses and every actor and critic
parameter gradient (the critic's = d critic_loss + d actor_loss).

`absolute=True` evaluates the same expression on absolute values (|W|, |b|, |x|, the ReLU
masks of the real evaluation, tanh and 1 - y^2 replaced by their absolute first-order
perturbation terms): the magnitude that rounding errors of a float32 evaluation scale with.
"""
import numpy as np


def _forward(layers, x, masks=None, absolute=False):
    """acts[l] = input of layer l, acts[-1] = head output; masks: the ReLU masks (computed on
    the real pass and reused by the absolute one)."""
    acts, own, pre = [x], [], []
    for l, (w, b) in enumerate(layers):
        z = x @ (np.abs(w) if absolute else w).T + (np.abs(b) if absolute else b)
        if l < len(layers) - 1:
            m = (z > 0) if masks is None else masks[l]
            own.append(m)
            pre.append(z)
            z = z * m
        acts.append(z)
        x = z
    return acts, own, pre


def _backward(layers, acts, masks, dout, absolute=False, input_grad=False):
    grads, d = [None] * len(layers), dout
    for l in reversed(range(len(layers))):
        w = np.abs(layers[l][0]) if absolute else layers[l][0]
        grads[l] = (d.T @ acts[l], d.sum(axis=0))
        if l > 0:
            d = (d @ w) * masks[l - 1]
        elif input_grad:
            d = d @ w
    return grads, d


def n_step_returns(rewards, done, qt, n_step, gamma, absolute=False):
    """rewards [C, E, Np], done [C, E] in time order, qt [valid, E, Np] the bootstrap value of
    each window (target critic at slot i + n_step; the last window: slot C - 1)."""
    valid = rewards.shape[0] - n_step + 1
    d = np.asarray(done, dtype=np.float64)[:, :, None]
    om = np.abs(1 - d) if absolute else 1 - d
    ret = np.empty((valid,) + rewards.shape[1:])
    for i in range(valid):
        last = i + n_step - 1
        if i < valid - 1:
            r = rewards[last] + om[last] * gamma * qt[i]
        else:
            r = (np.abs(d[last]) if absolute else d[last]) * rewards[last] + om[last] * qt[i]
        for j in range(1, n_step):
            k = n_step - 1 - j + i
            r = om[k] * gamma * r + rewards[k]
        ret[i] = r
    return ret


def ddpg_update(obs, actions, rewards, done, cursor, n_step, gamma, scale, bias, actor,
                critic, target_actor, target_critic, absolute=False, _real=None):
    """obs [C, E, Np, F], actions [C, E, Np, A], rewards [C, E, Np], done [C, E] in physical
    slot order, `cursor` the oldest slot; networks: [(W [out, in], b)], hidden layers then the
    head.  Returns a dict: values, j_values, returns [valid, E, Np], sum_sq_err, sum_j,
    critic_loss, actor_loss, actor_grads / critic_grads [(dW, db)] and, for the bound, the
    ReLU pre-activations of every network's hidden layers ("pre")."""
    if absolute and _real is None:
        _real = ddpg_update(obs, actions, rewards, done, cursor, n_step, gamma, scale, bias,
                            actor, critic, target_actor, target_critic)
    ab = (lambda v: np.abs(v)) if absolute else (lambda v: v)
    f64 = lambda v: np.asarray(v, dtype=np.float64)  # noqa: E731
    C, E, Np, F = obs.shape
    A = actions.shape[-1]
    order = (cursor + np.arange(C)) % C
    obs, actions = ab(f64(obs)[order]), ab(f64(actions)[order])
    rewards, done = ab(f64(rewards)[order]), f64(done)[order]
    scale, bias, gamma = float(scale), float(bias), float(gamma)
    valid = C - n_step + 1
    M = valid * E * Np
    tslot = [i + n_step if i < valid - 1 else C - 1 for i in range(valid)]
    o = obs[:valid].reshape(M, F)
    a = actions[:valid].reshape(M, A)
    ot = obs[tslot].reshape(M, F)
    R = _real or {}
    mk = R.get("masks", {})

    pre = {}

    def fwd(name, layers, x):
        acts, m, pre[name] = _forward(layers, x, mk.get(name), absolute)
        if not absolute:
            mk[name] = m
        return acts

    def head(acts, name):
        z = acts[-1]
        if absolute:
            y = np.abs(np.tanh(_real["z"][name]))
            return abs(scale) * (y + z) + abs(bias), y, z
        y = np.tanh(z)
        return scale * y + bias, y, z

    ta_acts = fwd("target_actor", target_actor, ot)
    at, _, zt = head(ta_acts, "target_actor")
    tc_acts = fwd("target_critic", target_critic, np.concatenate([ot, at], axis=1))
    qt = tc_acts[-1][:, 0].reshape(valid, E, Np)

    ret = n_step_returns(rewards, done, qt, n_step, gamma, absolute)

    q_acts = fwd("critic_q", critic, np.concatenate([o, a], axis=1))
    a_acts = fwd("actor", actor, o)
    pi, y, z = head(a_acts, "actor")
    j_acts = fwd("critic_j", critic, np.concatenate([o, pi], axis=1))
    values = q_acts[-1][:, 0].reshape(valid, E, Np)
    j_values = j_acts[-1][:, 0].reshape(valid, E, Np)

    diff = (values + ret) if absolute else (values - ret)
    dq = (2.0 / M) * diff.reshape(M, 1)
    dj = np.full((M, 1), -1.0 / M)
    if absolute:
        dj = np.abs(dj)
    gq, _ = _backward(critic, q_acts, mk["critic_q"], dq, absolute)
    gj, dx = _backward(critic, j_acts, mk["critic_j"], dj, absolute, input_grad=True)
    dpi = dx[:, F:]
    if absolute:
        yr = _real["y"]
        dz = abs(scale) * dpi * (1 + yr * yr + 2 * np.abs(yr) * (y + z))
    else:
        dz = scale * dpi * (1 - y * y)
    ga, _ = _backward(actor, a_acts, mk["actor"], dz, absolute)
    critic_grads = [(gq[l][0] + gj[l][0], gq[l][1] + gj[l][1]) for l in range(len(critic))]
    out = {
        "values": values, "j_values": j_values, "returns": ret,
        "sum_sq_err": float((diff ** 2).sum()), "sum_j": float(j_values.sum()),
        "critic_loss": float((diff ** 2).sum() / M), "actor_loss": float(-j_values.sum() / M),
        "actor_grads": ga, "critic_grads": critic_grads, "pre": pre,
    }
    if not absolute:
        out["masks"] = mk
        out["z"] = {"target_actor": zt, "actor": z}
        out["y"] = y
    return out
