"""Float64 reference of the five sampled-row update passes (wdb_*_update_sampled,
include/wdb200.h): the windows gathered by index from the physical ring, the sampled n-step
return as a NumPy recursion, and the losses on the project's own networks cast to float64, with
every gradient by torch autograd.  Row g of every result belongs to windows[g]."""
import copy

import numpy as np
import torch


def gather(ring, windows, n_step, n_agents):
    """ring = (obs [C, E, Np, F], actions [C, E, Np, A], rewards [C, E, Np], done [C, E]) in
    physical slot order, windows int [B, 2] (start slot, agent row) -> float64 obs [B, F],
    actions [B, A], rewards [n_step, B], done [n_step, B], bootstrap obs [B, F]."""
    obs, actions, rewards, done = (np.asarray(r, dtype=np.float64) for r in ring)
    C = obs.shape[0]
    windows = np.asarray(windows, dtype=np.int64)
    start, row = windows[:, 0], windows[:, 1]
    assert ((0 <= start) & (start < C)).all() and ((0 <= row) & (row < rewards[0].size)).all()
    steps = (start[None, :] + np.arange(n_step + 1)[:, None]) % C
    obs = obs.reshape(C, -1, obs.shape[-1])
    return (obs[start, row], actions.reshape(C, -1, actions.shape[-1])[start, row],
            rewards.reshape(C, -1)[steps[:-1], row], done[steps[:-1], row // n_agents],
            obs[steps[-1], row])


def sampled_returns(rewards, done, boot, gamma):
    """R = r_0 + (1 - d_0) gamma (r_1 + ... (1 - d_{n-1}) gamma boot): rewards, done [n, B]."""
    r = np.asarray(boot, dtype=np.float64)
    for j in reversed(range(rewards.shape[0])):
        r = (1.0 - done[j]) * gamma * r + rewards[j]
    return r


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


def _grads(loss, *models):
    params = [p for m in models for p in m.parameters()]
    return [g.numpy() for g in torch.autograd.grad(loss, params, retain_graph=True)]


def _f64(models):
    return [copy.deepcopy(m).cpu().double() for m in models]


def ddpg_sampled(models, ring, windows, n_step, gamma):
    """models = (actor, critic, target_actor, target_critic).  Gradients in parameter order:
    the actor's = d actor_loss, the critic's = d critic_loss + d actor_loss."""
    actor, critic, t_actor, t_critic = _f64(models)
    n_agents = ring[2].shape[2]
    obs, actions, rewards, done, boot_obs = gather(ring, windows, n_step, n_agents)
    with torch.no_grad():
        boot = t_critic(obs=_t(boot_obs), action=t_actor(obs=_t(boot_obs))).numpy()
    returns = sampled_returns(rewards, done, boot, gamma)
    values = critic(obs=_t(obs), action=_t(actions))
    j_values = critic(obs=_t(obs), action=actor(obs=_t(obs)))
    err = values - _t(returns)
    loss = (err ** 2).mean() - j_values.mean()
    return {"values": values.detach().numpy(), "j_values": j_values.detach().numpy(),
            "returns": returns, "sum_sq_err": float((err ** 2).sum().detach()),
            "sum_j": float(j_values.sum().detach()), "actor_grads": _grads(-j_values.mean(), actor),
            "critic_grads": _grads(loss, critic)}


def td3_critic_sampled(algo, models, ring, windows, noise, n_step, gamma):
    """models = (target_actor, target_critic, target_critic2, critic, critic2)."""
    t_actor, t_c1, t_c2, c1, c2 = _f64(models)
    n_agents = ring[2].shape[2]
    obs, actions, rewards, done, boot_obs = gather(ring, windows, n_step, n_agents)
    with torch.no_grad():
        pi = torch.cat(list(t_actor(obs=_t(boot_obs))), dim=-1)
        a_t = algo.target_actions(pi, _t(np.asarray(noise, dtype=np.float64)),
                                  float(t_actor.action_scale), float(t_actor.action_bias))
        boot = torch.minimum(t_c1(obs=_t(boot_obs), action=a_t),
                             t_c2(obs=_t(boot_obs), action=a_t)).numpy()
    returns = sampled_returns(rewards, done, boot, gamma)
    q1, q2 = c1(obs=_t(obs), action=_t(actions)), c2(obs=_t(obs), action=_t(actions))
    e1, e2 = q1 - _t(returns), q2 - _t(returns)
    loss = (e1 ** 2).mean() + (e2 ** 2).mean()
    return {"q1": q1.detach().numpy(), "q2": q2.detach().numpy(), "returns": returns,
            "sums": (float((e1 ** 2).sum().detach()), float((e2 ** 2).sum().detach())),
            "critic_grads": _grads(loss, c1), "critic2_grads": _grads(loss, c2)}


def td3_actor_sampled(models, ring, windows, n_step):
    """models = (actor, critic); the gradient of -mean Q1(obs, actor(obs)) wrt the actor."""
    actor, critic = _f64(models)
    obs = gather(ring, windows, n_step, ring[2].shape[2])[0]
    j = critic(obs=_t(obs), action=actor(obs=_t(obs)))
    return {"j_values": j.detach().numpy(), "sum_j": float(j.sum().detach()),
            "actor_grads": _grads(-j.mean(), actor)}


def sac_critic_sampled(models, log_alpha, ring, windows, noise, n_step, gamma):
    """models = (actor, target_critic, target_critic2, critic, critic2)."""
    actor, t_c1, t_c2, c1, c2 = _f64(models)
    n_agents = ring[2].shape[2]
    obs, actions, rewards, done, boot_obs = gather(ring, windows, n_step, n_agents)
    with torch.no_grad():
        a_t, log_pi = actor.sample(_t(boot_obs), _t(np.asarray(noise, dtype=np.float64)))
        q_t = torch.minimum(t_c1(obs=_t(boot_obs), action=a_t), t_c2(obs=_t(boot_obs), action=a_t))
        boot = (q_t - float(np.exp(log_alpha)) * log_pi).numpy()
    returns = sampled_returns(rewards, done, boot, gamma)
    q1, q2 = c1(obs=_t(obs), action=_t(actions)), c2(obs=_t(obs), action=_t(actions))
    e1, e2 = q1 - _t(returns), q2 - _t(returns)
    loss = (e1 ** 2).mean() + (e2 ** 2).mean()
    return {"q1": q1.detach().numpy(), "q2": q2.detach().numpy(), "returns": returns,
            "sums": (float((e1 ** 2).sum().detach()), float((e2 ** 2).sum().detach())),
            "critic_grads": _grads(loss, c1), "critic2_grads": _grads(loss, c2)}


def sac_actor_sampled(models, log_alpha, ring, windows, noise, n_step):
    """models = (actor, critic, critic2); mean(alpha log pi - min(Q1, Q2)), ties to Q1."""
    actor, c1, c2 = _f64(models)
    obs = gather(ring, windows, n_step, ring[2].shape[2])[0]
    a, log_pi = actor.sample(_t(obs), _t(np.asarray(noise, dtype=np.float64)))
    q1, q2 = c1(obs=_t(obs), action=a), c2(obs=_t(obs), action=a)
    q = torch.where(q1 <= q2, q1, q2)
    loss = (float(np.exp(log_alpha)) * log_pi - q).mean()
    return {"log_probs": log_pi.detach().numpy(),
            "sums": (float(q.sum().detach()), float(log_pi.sum().detach())), "actor_grads": _grads(loss, actor)}
