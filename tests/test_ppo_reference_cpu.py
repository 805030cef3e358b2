"""The float64 reference of the multi-epoch PPO kernels (ppo_reference.py) against torch autograd
in float64, without a GPU: GAE against the policy-gradient module's CPU branch (and, at
lambda = 1, against the existing discounted returns), the clipped loss and every gradient
(probabilities, mean, log_std, values) against `ppo_minibatch_loss` -- the float32 torch
expression the trainer falls back to -- evaluated in float64.  The cases include ties of the
minimum, rho exactly on the clip boundary, zero advantages, probabilities on the Categorical
clamp boundary and masked (zero-probability) actions."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import ppo_reference as ref  # noqa: E402

EPS64 = 2.0 ** -52
TOL = 1e-12


def _close(got, want, tol=TOL):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    err = np.abs(got - want) / np.maximum(1.0, np.abs(want))
    assert (err <= tol).all(), float(err.max())


def _episode_inputs(T, E, Np, seed, p_done):
    rng = np.random.default_rng(seed)
    r = rng.normal(size=(T, E, Np))
    v = rng.normal(size=(T, E, Np))
    d = (rng.random((T, E)) < p_done).astype(np.int32) * rng.integers(1, 3, (T, E))
    return r, v, d


@pytest.mark.parametrize("lam", [0.0, 0.5, 0.95, 1.0])
@pytest.mark.parametrize("p_done", [0.0, 0.2, 1.0])
def test_gae_reference_equals_the_module_cpu_branch(lam, p_done):
    from warp_drive_b200.training.algorithms.policygradient import gae

    r, v, d = _episode_inputs(9, 7, 3, seed=int(lam * 100) + int(p_done * 10), p_done=p_done)
    adv, vt = ref.gae(r, v, d, 0.97, lam)
    ta, tv = gae(torch.from_numpy(r), torch.from_numpy(d), torch.from_numpy(v),
                 float(np.float32(0.97)), float(np.float32(lam)))
    _close(ta.numpy(), adv[0], 1e-11)
    _close(tv.numpy(), vt[0], 1e-11)


@pytest.mark.parametrize("p_done", [0.0, 0.3, 1.0])
def test_gae_at_lambda_one_is_the_discounted_return(p_done):
    from warp_drive_b200.training.algorithms.policygradient import discounted_returns

    r, v, d = _episode_inputs(12, 5, 2, seed=4, p_done=p_done)
    gamma = float(np.float32(0.95))
    _, vt = ref.gae(r, v, d, gamma, 1.0)
    ret = discounted_returns(torch.from_numpy(r), torch.from_numpy(d), torch.from_numpy(v), gamma)
    _close(vt[0], ret.numpy())


def test_gae_at_lambda_zero_is_one_step_td():
    r, v, d = _episode_inputs(6, 4, 1, seed=8, p_done=0.0)
    gamma = float(np.float32(0.9))
    adv, vt = ref.gae(r, v, d, gamma, 0.0)
    _close(vt[0][:-1], r[:-1] + gamma * v[1:])


# ---------------------------------------------------------------------------- the loss
def _cat_case(B, widths, seed, clip):
    """Categorical rows with every boundary case: dyadic rows whose z and q are exact, rows on
    the float64 clamp boundary (q = eps and 1 - eps), masked actions (p = 0), zero advantages,
    rho == 1 exactly (old = l) and rho spread across the clip interval."""
    rng = np.random.default_rng(seed)
    probs, actions = [], []
    for A in widths:
        p = rng.random((B, A)) + 0.05
        if A >= 2:
            p[::5, 0] = 0.0                                     # masked action
            p[1::5] = 0.0
            p[1::5, 0], p[1::5, 1] = 1.0 - EPS64, EPS64             # on the clamp boundary
            p[2::5] = 0.0
            p[2::5, 0], p[2::5, 1] = 0.5, 0.5                       # dyadic: exact z and q
        a = rng.integers(0, A, B)
        a[::5] = np.where(A > 1, 1 + (a[::5] % max(A - 1, 1)), 0)
        a[::5] = np.minimum(a[::5], A - 1)
        probs.append(p)
        actions.append(a)
    actions = np.stack(actions, -1)
    values = rng.normal(size=B)
    adv = rng.normal(size=B)
    adv[3::7] = 0.0
    vt = rng.normal(size=B)
    return probs, values, actions, adv, vt


def _torch_cat(probs, values, actions, adv, vt, old, ppo, clip, vf, ent):
    from warp_drive_b200.training.algorithms.policygradient import ppo_minibatch_loss

    P = [torch.tensor(p, dtype=torch.float64, requires_grad=True) for p in probs]
    V = torch.tensor(values, dtype=torch.float64, requires_grad=True)
    loss, sums = ppo_minibatch_loss(P, V, torch.from_numpy(actions), torch.from_numpy(adv),
                                    torch.from_numpy(vt), torch.from_numpy(old), ppo, clip, vf,
                                    ent)
    loss.backward()
    return loss, sums, [p.grad.numpy() for p in P], V.grad.numpy()


def _logp64(probs, actions):
    from torch.distributions import Categorical

    return sum(Categorical(torch.from_numpy(p)).log_prob(torch.from_numpy(actions[:, k]))
               for k, p in enumerate(probs)).numpy()


@pytest.mark.parametrize("widths", [[3], [2, 5], [4, 1, 7, 2]])
@pytest.mark.parametrize("ppo,clip", [(True, 0.2), (True, 0.0), (False, 0.2)])
def test_categorical_loss_reference_equals_torch_autograd_in_float64(widths, ppo, clip):
    B = 60
    probs, values, actions, adv, vt = _cat_case(B, widths, seed=len(widths), clip=clip)
    logp = _logp64(probs, actions)
    vf, ent = 0.7, 0.03
    rng = np.random.default_rng(5)
    old = logp + rng.uniform(-0.5, 0.5, B)
    # rho == 1 exactly on every fourth row (a tie of the minimum; with clip 0 also both ends of
    # the interval): each side gets its own log-prob there (the reference multiplies by 1 / z
    # as the kernel does, torch divides: they may differ in the last bit)
    old_r = old.copy()
    old_r[::4] = ref.ppo_loss(probs, values, actions, adv, vt, old, ppo, clip, vf, ent,
                              prob_eps=EPS64)["logp"][0][::4]
    old[::4] = logp[::4]
    r = ref.ppo_loss(probs, values, actions, adv, vt, old_r, ppo, clip, vf, ent, prob_eps=EPS64)
    _close(r["logp"][0], logp)
    assert (r["rho"][0][::4] == 1.0).all()
    loss, sums, g_probs, g_values = _torch_cat(probs, values, actions, adv, vt, old, ppo, clip,
                                               vf, ent)
    for got, want in zip(g_probs, r["grad_probs"]):
        _close(got, want[0])
    _close(g_values, r["grad_values"][0])
    for k in range(4):
        _close(float(sums[k]), r["sums"][k][0])
    assert int(sums[4]) == r["sums"][4][0]
    _close(float(loss.detach()), ref.loss_value(r["sums"], B, vf, ent)[0])


def test_categorical_boundary_rows_take_torch_branches():
    """The clamp boundary passes the gradient (both ends inclusive), a masked action gets the
    entropy term only, and at rho == 1 with clip 0 (rho on both ends of the interval) the
    minimum's tie hands the full advantage to the log-prob."""
    probs = [np.array([[1.0 - EPS64, EPS64, 0.0], [0.5, 0.5, 0.0]])]   # z and q exact
    actions = np.array([[1], [0]])
    logp = _logp64(probs, actions)
    adv, values, vt = np.array([0.7, -1.3]), np.array([0.1, 0.2]), np.array([0.0, 0.5])
    r = ref.ppo_loss(probs, values, actions, adv, vt, logp, True, 0.0, 0.5, 0.01, prob_eps=EPS64)
    assert (r["rho"][0] == 1.0).all()
    _, _, g_probs, _ = _torch_cat(probs, values, actions, adv, vt, logp, True, 0.0, 0.5, 0.01)
    _close(g_probs[0], r["grad_probs"][0][0])
    # the a2c weight on the taken action: -adv / (B q) from the log-prob term
    a2c = ref.ppo_loss(probs, values, actions, adv, vt, logp, False, 0.0, 0.5, 0.01,
                       prob_eps=EPS64)
    _close(r["grad_probs"][0][0], a2c["grad_probs"][0][0])


def _gauss_case(B, A, seed):
    rng = np.random.default_rng(seed)
    mean = rng.normal(size=(B, A))
    log_std = 0.4 * rng.normal(size=A)
    actions = mean + np.exp(log_std) * rng.normal(size=(B, A))
    values, adv, vt = rng.normal(size=B), rng.normal(size=B), rng.normal(size=B)
    adv[2::6] = 0.0
    return mean, log_std, values, actions, adv, vt


@pytest.mark.parametrize("A", [1, 3, 8])
@pytest.mark.parametrize("ppo,clip", [(True, 0.2), (True, 0.0), (False, 0.2)])
def test_gaussian_loss_reference_equals_torch_autograd_in_float64(A, ppo, clip):
    from warp_drive_b200.training.algorithms.policygradient import ppo_minibatch_loss

    B = 50
    mean, log_std, values, actions, adv, vt = _gauss_case(B, A, seed=A)
    r0 = ref.ppo_gaussian_loss(mean, log_std, values, actions, adv, vt, np.zeros(B), ppo, clip,
                               0.5, 0.02, float64=True)
    old = r0["logp"][0] + np.random.default_rng(1).uniform(-0.4, 0.4, B)
    old_r = old.copy()
    old_r[::3] = r0["logp"][0][::3]                         # rho == 1 exactly, on each side
    r = ref.ppo_gaussian_loss(mean, log_std, values, actions, adv, vt, old_r, ppo, clip, 0.5,
                              0.02, float64=True)
    assert (r["rho"][0][::3] == 1.0).all()
    with torch.no_grad():
        from torch.distributions import Normal

        lt = Normal(torch.from_numpy(mean), torch.from_numpy(log_std).exp()).log_prob(
            torch.from_numpy(actions)).sum(-1).numpy()
    _close(lt, r0["logp"][0])
    old[::3] = lt[::3]
    mu = torch.tensor(mean, requires_grad=True)
    ls = torch.tensor(log_std, requires_grad=True)
    V = torch.tensor(values, requires_grad=True)
    loss, sums = ppo_minibatch_loss([mu], V, torch.from_numpy(actions), torch.from_numpy(adv),
                                    torch.from_numpy(vt), torch.from_numpy(old), ppo, clip, 0.5,
                                    0.02, log_std=ls)
    loss.backward()
    _close(mu.grad.numpy(), r["grad_mean"][0])
    _close(ls.grad.numpy(), r["grad_log_std"][0])
    _close(V.grad.numpy(), r["grad_values"][0])
    for k in range(4):
        _close(float(sums[k]), r["sums"][k][0])
    assert int(sums[4]) == r["sums"][4][0]
    _close(float(loss.detach()), ref.loss_value(r["sums"], B, 0.5, 0.02)[0])
