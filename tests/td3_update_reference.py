"""Float64 NumPy restatement of one TD3 update of one policy -- what `wdb_td3_critic_update`
and `wdb_td3_actor_update` compute (include/wdb200.h) and what TrainerTD3's torch update
computes by autograd (algorithms/td3.py): the critic pass (target actor + clipped noise, both
target critics, their minimum, the n-step return, both critic losses and both critics'
gradients) and the actor pass (-mean Q1(s, pi(s)) and the actor's gradient).

`absolute=True` evaluates the same expressions on absolute values (as ddpg_update_reference
does): the magnitude that rounding errors of a float32 evaluation scale with.  The clamps and
the minimum are taken from the real evaluation and applied to the absolute one (a clamped
noise or action contributes its bound, which carries no rounding of the inputs).
"""
import numpy as np

from ddpg_update_reference import _backward, _forward, n_step_returns


def _prep(obs, actions, rewards, done, cursor, n_step, absolute):
    f64 = lambda v: np.asarray(v, dtype=np.float64)  # noqa: E731
    ab = np.abs if absolute else (lambda v: v)
    C = obs.shape[0]
    order = (cursor + np.arange(C)) % C
    return (ab(f64(obs)[order]), ab(f64(actions)[order]), ab(f64(rewards)[order]),
            f64(done)[order])


def td3_critic_update(obs, actions, rewards, done, cursor, n_step, gamma, scale, bias, sigma,
                      clip, noise, critic, critic2, target_actor, target_critic, target_critic2,
                      absolute=False, _real=None):
    """obs [C, E, Np, F], actions [C, E, Np, A], rewards [C, E, Np], done [C, E] in physical
    slot order, `cursor` the oldest slot; noise [valid, E, Np, A]; networks [(W [out, in], b)],
    hidden layers then the head.  Returns q1 / q2 / returns [valid, E, Np], sum_sq_err1 / 2,
    critic1_loss / critic2_loss, critic_grads / critic2_grads [(dW, db)], "pre" (ReLU
    pre-activations) and, for the cases, which clamps and which critic the minimum hit."""
    if absolute and _real is None:
        _real = td3_critic_update(obs, actions, rewards, done, cursor, n_step, gamma, scale,
                                  bias, sigma, clip, noise, critic, critic2, target_actor,
                                  target_critic, target_critic2)
    obs, actions, rewards, done = _prep(obs, actions, rewards, done, cursor, n_step, absolute)
    scale, bias, gamma = float(scale), float(bias), float(gamma)
    C, E, Np, F = obs.shape
    A = actions.shape[-1]
    valid = C - n_step + 1
    M = valid * E * Np
    tslot = [i + n_step if i < valid - 1 else C - 1 for i in range(valid)]
    o, a = obs[:valid].reshape(M, F), actions[:valid].reshape(M, A)
    ot = obs[tslot].reshape(M, F)
    eps = np.asarray(noise, dtype=np.float64).reshape(M, A)
    R = _real or {}
    mk = R.get("masks", {})
    pre = {}

    def fwd(name, layers, x):
        acts, m, pre[name] = _forward(layers, x, mk.get(name), absolute)
        if not absolute:
            mk[name] = m
        return acts

    zt = fwd("target_actor", target_actor, ot)[-1]
    if absolute:
        # pi' = scale tanh(z) + bias, then + noise: first-order terms of each rounding;
        # clamped entries are the bound itself
        y = np.abs(np.tanh(R["zt"]))
        pi = abs(scale) * (y + zt) + abs(bias)
        nz = np.where(R["noise_clamped"], abs(clip * scale), abs(sigma * scale) * np.abs(eps))
        at = np.where(R["action_clamped"], abs(bias) + abs(scale), pi + nz)
    else:
        pi = scale * np.tanh(zt) + bias
        raw = sigma * scale * eps
        nz = np.clip(raw, -clip * scale, clip * scale)
        pre_a = pi + nz
        at = np.clip(pre_a, bias - scale, bias + scale)
    x_t = np.concatenate([ot, at], axis=1)
    qt1 = fwd("target_critic", target_critic, x_t)[-1][:, 0]
    qt2 = fwd("target_critic2", target_critic2, x_t)[-1][:, 0]
    if absolute:
        first = R["min_is_first"]
    else:
        first = qt1 <= qt2
    qt = np.where(first, qt1, qt2).reshape(valid, E, Np)
    ret = n_step_returns(rewards, done, qt, n_step, gamma, absolute)

    q1_acts = fwd("critic_q1", critic, np.concatenate([o, a], axis=1))
    q2_acts = fwd("critic_q2", critic2, np.concatenate([o, a], axis=1))
    q1 = q1_acts[-1][:, 0].reshape(valid, E, Np)
    q2 = q2_acts[-1][:, 0].reshape(valid, E, Np)
    d1 = (q1 + ret) if absolute else (q1 - ret)
    d2 = (q2 + ret) if absolute else (q2 - ret)
    g1, _ = _backward(critic, q1_acts, mk["critic_q1"], (2.0 / M) * d1.reshape(M, 1), absolute)
    g2, _ = _backward(critic2, q2_acts, mk["critic_q2"], (2.0 / M) * d2.reshape(M, 1), absolute)
    out = {
        "q1": q1, "q2": q2, "returns": ret,
        "sum_sq_err1": float((d1 ** 2).sum()), "sum_sq_err2": float((d2 ** 2).sum()),
        "critic1_loss": float((d1 ** 2).sum() / M), "critic2_loss": float((d2 ** 2).sum() / M),
        "critic_grads": g1, "critic2_grads": g2, "pre": pre,
    }
    if not absolute:
        out.update(masks=mk, zt=zt, min_is_first=first,
                   noise_clamped=np.abs(raw) > clip * scale,
                   action_clamped=(pre_a < bias - scale) | (pre_a > bias + scale))
    return out


def td3_actor_update(obs, cursor, n_step, scale, bias, actor, critic, absolute=False,
                     _real=None):
    """The actor pass on the same ring: J = Q1(s, pi(s)) [valid, E, Np], sum_j, actor_loss
    and actor_grads [(dW, db)]."""
    if absolute and _real is None:
        _real = td3_actor_update(obs, cursor, n_step, scale, bias, actor, critic)
    C, E, Np, F = obs.shape
    order = (cursor + np.arange(C)) % C
    obs = np.asarray(obs, dtype=np.float64)[order]
    if absolute:
        obs = np.abs(obs)
    scale, bias = float(scale), float(bias)
    valid = C - n_step + 1
    M = valid * E * Np
    o = obs[:valid].reshape(M, F)
    R = _real or {}
    mk = R.get("masks", {})
    pre = {}

    def fwd(name, layers, x):
        acts, m, pre[name] = _forward(layers, x, mk.get(name), absolute)
        if not absolute:
            mk[name] = m
        return acts

    a_acts = fwd("actor", actor, o)
    z = a_acts[-1]
    if absolute:
        y = np.abs(np.tanh(R["z"]))
        pi = abs(scale) * (y + z) + abs(bias)
    else:
        y = np.tanh(z)
        pi = scale * y + bias
    j_acts = fwd("critic_j", critic, np.concatenate([o, pi], axis=1))
    j = j_acts[-1][:, 0].reshape(valid, E, Np)
    dj = np.full((M, 1), (1.0 if absolute else -1.0) / M)
    _, dx = _backward(critic, j_acts, mk["critic_j"], dj, absolute, input_grad=True)
    dpi = dx[:, F:]
    if absolute:
        yr = np.tanh(R["z"])
        dz = abs(scale) * dpi * (1 + yr * yr + 2 * np.abs(yr) * (y + z))
    else:
        dz = scale * dpi * (1 - y * y)
    ga, _ = _backward(actor, a_acts, mk["actor"], dz, absolute)
    out = {"j_values": j, "sum_j": float(j.sum()), "actor_loss": float(-j.sum() / M),
           "actor_grads": ga, "pre": pre}
    if not absolute:
        out.update(masks=mk, z=z)
    return out
