"""tests/sac_update_bounds.py on the CPU: its values are those of the float64 references of the
SAC-family passes (replay_update_reference.sac_*_sampled, sac_discrete_reference,
tqc_reference), a float32 torch evaluation of each pass through the algorithm classes (SAC,
DiscreteSAC, TQC and their torch losses: other operations and orders than the kernels') lies
within its bars, and its per-element bars reject small defects that a norm-wise 2e-4 check
accepts.  The case builder here feeds tests/test_gpu_sac_family_exact.py too."""
import copy
import math

import numpy as np
import pytest
import torch

import dqn_update_reference as dref
import replay_update_reference as rref
import sac_discrete_reference as dsref
import sac_update_bounds as sb
import tqc_reference as tref
from test_gpu_tqc import _Net
from test_q_update_bounds_cpu import within

LN_ALPHA = math.log(0.3)


def _layers64(model):
    from warp_drive_b200.training.algorithms.fused_ddpg import _layers

    return [(w.detach().double().cpu().numpy(), b.detach().double().cpu().numpy())
            for w, b in _layers(model)]


def make_models(kind, F, A, ad, cd, N=1, lo=-5.0, hi=1.0, scale=2.0, bias=0.25, seed=0):
    """Float32 (actor, critic, critic2, target_critic, target_critic2) as the fused wrappers read
    them (tests/test_gpu_tqc.py's _Net: no hidden layer allowed); the targets differ."""
    torch.manual_seed(seed)
    if kind == "discrete":
        actor = _Net(F, ad, A, "policy_head", flattened_obs_size=F, output_dims=[A])
        critics = [_Net(F, cd, A, "policy_head", flattened_obs_size=F, output_dims=[A])
                   for _ in range(4)]
    else:
        actor = _Net(F, ad, 2 * A, "policy_head", flattened_obs_size=F, output_dims=[A],
                     log_std_min=lo, log_std_max=hi, action_scale=scale, action_bias=bias)
        out = N if kind == "tqc" else 1
        critics = [_Net(F + A, cd, out, "vf_head", num_quantiles=N, flattened_obs_size=F)
                   for _ in range(4)]
    return [m.float() for m in [actor] + critics]


class Case:
    """One SAC-family pass pair on one shape: float32 models, a ring, B windows whose every
    premise holds in both passes (one wraps the ring's physical end, one is a duplicate), the
    noise rows (eps', eps), and the bar references.

    kind: "sac", "discrete" or "tqc".  done_vals: the done flags drawn in the ring.
    noise_scale multiplies the normals (|u| > 10 with a large one); log_std_bias shifts the raw
    log-std columns of the actor's head (the clamp's sides); pin: head rows of the raw log-std
    set to a constant lo or hi by zeroed weights (pinned to the clamp); ties: TQC target heads
    made near-tied ("exact": all atoms equal, "ulp": a few ulp apart, "straddle": critic 2's
    atoms interleave critic 1's around the cutoff)."""

    def __init__(self, kind, B, n_step, C, E, Np, F, A, ad, cd, gamma=0.97, N=1, d=0,
                 log_alpha=LN_ALPHA, lo=-5.0, hi=1.0, scale=2.0, bias=0.25, noise_scale=1.0,
                 log_std_bias=0.0, pin=None, ties=None, done_vals=(0, 1), seed=None,
                 models=None):
        seed = B + 7 * F + A if seed is None else seed
        self.kind, self.B, self.n_step, self.C, self.E, self.Np = kind, B, n_step, C, E, Np
        self.F, self.A, self.N, self.d = F, A, N, d
        self.gamma = float(np.float32(gamma))
        self.log_alpha = float(np.float32(log_alpha))
        self.lo, self.hi = float(np.float32(lo)), float(np.float32(hi))
        self.scale, self.bias = float(np.float32(scale)), float(np.float32(bias))
        if models is None:
            models = make_models(kind, F, A, ad, cd, N, lo, hi, scale, bias, seed)
            self._shape(models, log_std_bias, pin, ties)
        self.models = models
        g = np.random.default_rng(seed)
        obs = g.standard_normal((C, E, Np, F)).astype(np.float32)
        if kind == "discrete":
            actions = g.integers(0, A, (C, E, Np, 1)).astype(np.int32)
        else:
            actions = g.uniform(-2.0, 2.0, (C, E, Np, A)).astype(np.float32)
        rewards = g.standard_normal((C, E, Np)).astype(np.float32)
        done = np.asarray(done_vals, np.int32)[g.integers(0, len(done_vals), (C, E))]
        done[g.random((C, E)) < 0.6] = 0
        self.ring = [obs, actions, rewards, done]
        n = B + B // 2 + 64
        w = np.stack([g.integers(0, C, n), g.integers(0, E * Np, n)], axis=1).astype(np.int32)
        w[0] = (C - 1, E * Np - 1)                      # wraps the physical end of the ring
        noise = (noise_scale * g.standard_normal((2, n, A))).astype(np.float32)
        self.windows, self.noise_c, self.noise_a = w, noise[0], noise[1]
        refs = self.reference()
        keep = np.flatnonzero(refs[0]["ok"] & refs[1]["ok"])
        if len(keep) < B:
            pytest.fail(f"only {len(keep)} of {n} drawn windows satisfy every premise; {B} needed")
        keep = keep[:B].copy()
        if B > 2:
            keep[2] = keep[1]                            # a duplicate window (and its noise)
        self.windows = w[keep].copy()
        self.noise_c, self.noise_a = noise[0][keep].copy(), noise[1][keep].copy()

    def _shape(self, models, log_std_bias, pin, ties):
        actor = models[0]
        A = self.A
        with torch.no_grad():
            if self.kind != "discrete":
                actor.policy_head.bias[A:] += log_std_bias
                if pin is not None:                  # raw log-std columns pinned to lo or hi
                    for c, v in pin:
                        actor.policy_head.weight[A + c].zero_()
                        actor.policy_head.bias[A + c] = v
            for t in models[3:]:
                for p in t.parameters():
                    p.add_(0.3 * torch.randn_like(p))
            if ties is not None:
                t1, t2 = models[3].vf_head, models[4].vf_head
                N = self.N
                for t in (t1, t2):
                    t.weight.mul_(1e-3 if ties != "exact" else 0.0)
                if ties == "exact":
                    t1.bias.fill_(0.5)
                    t2.bias.fill_(0.5)
                elif ties == "ulp":                  # atoms a few ulp of 0.5 apart
                    ulp = float(np.spacing(np.float32(0.5)))
                    t1.bias.copy_(torch.tensor(0.5 + ulp * (np.arange(N) % 4)))
                    t2.bias.copy_(torch.tensor(0.5 + ulp * ((np.arange(N) + 1) % 3)))
                else:                                # interleaved across the two critics
                    base = np.linspace(0.0, 1.0, N)
                    t1.bias.copy_(torch.tensor(base))
                    t2.bias.copy_(torch.tensor(base + 0.5 / max(N - 1, 1) + 1e-6))

    # -------------------------------------------------------------- references
    def layers(self):
        return [_layers64(m) for m in self.models]

    def rows(self, w=None):
        w = self.windows if w is None else w
        if self.kind == "discrete":
            ring = [self.ring[0], self.ring[1][..., 0], self.ring[2], self.ring[3]]
            return dref.gather(ring, w, self.n_step, self.Np)
        return rref.gather(self.ring, w, self.n_step, self.Np)

    def reference(self):
        """(critic pass, actor pass) dicts of (value, bar)."""
        La, L1, L2, T1, T2 = self.layers()
        rows = self.rows()
        obs = rows[0]
        sq = dict(scale=self.scale, bias=self.bias, lo=self.lo, hi=self.hi)
        if self.kind == "sac":
            return (sb.sac_critic(La, L1, L2, T1, T2, rows, self.noise_c, self.gamma,
                                  self.log_alpha, **sq),
                    sb.sac_actor(La, L1, L2, obs, self.noise_a, self.log_alpha, **sq))
        if self.kind == "discrete":
            return (sb.sac_discrete_critic(La, L1, L2, T1, T2, rows, self.gamma, self.log_alpha),
                    sb.sac_discrete_actor(La, L1, L2, obs, self.log_alpha))
        return (sb.tqc_critic(La, L1, L2, T1, T2, rows, self.noise_c, self.gamma,
                              self.log_alpha, N=self.N, n_drop=self.d, **sq),
                sb.tqc_actor(La, L1, L2, obs, self.noise_a, self.log_alpha, N=self.N, **sq))

    @property
    def alpha(self):
        return math.exp(self.log_alpha)

    def existing(self):
        """The existing float64 references' (critic, actor) dicts on the same inputs."""
        La, L1, L2, T1, T2 = self.layers()
        ring64 = [r.astype(np.float64) if r.dtype == np.float32 else r for r in self.ring]
        w = self.windows
        if self.kind == "discrete":
            ring64[1] = ring64[1][..., 0]
            return (dsref.critic_pass(La, L1, L2, T1, T2, ring64, w, self.n_step, self.gamma,
                                      self.alpha),
                    dsref.actor_pass(La, L1, L2, ring64, w, self.n_step, self.alpha, 0.0))
        sq = dict(scale=self.scale, bias=self.bias, lo=self.lo, hi=self.hi)
        nc, na = self.noise_c.astype(np.float64), self.noise_a.astype(np.float64)
        if self.kind == "tqc":
            return (tref.critic_pass(La, [L1, L2], [T1, T2], ring64, w, self.n_step, self.gamma,
                                     self.alpha, noise=nc, n_drop=self.d, **sq),
                    tref.actor_pass(La, [L1, L2], ring64, w, self.n_step, self.alpha, noise=na,
                                    target_entropy=0.0, **sq))
        actor, c1, c2, t1, t2 = (_as_sac(m) for m in self.models)
        return (rref.sac_critic_sampled((actor, t1, t2, c1, c2), self.log_alpha, ring64, w, nc,
                                        self.n_step, self.gamma),
                rref.sac_actor_sampled((actor, c1, c2), self.log_alpha, ring64, w, na,
                                       self.n_step))


class _SacActor(torch.nn.Module):
    """A _Net actor with FullyConnectedSACActor's sample(): what replay_update_reference calls."""

    def __init__(self, net):
        super().__init__()
        self.net = net
        f32 = lambda v: float(np.float32(v))  # noqa: E731  the float32 values the kernels read
        self.lo, self.hi = f32(net.log_std_min), f32(net.log_std_max)
        self.scale, self.bias = f32(net.action_scale), f32(net.action_bias)

    def forward(self, obs):
        x = obs
        for i in range(len(self.net.fc)):
            x = self.net.fc[str(i)](x)
        return self.net.policy_head(x)

    def sample(self, obs, eps):
        from warp_drive_b200.training.models.fully_connected_actor_critic import (
            squashed_log_prob)

        z = self(obs)
        A = z.shape[-1] // 2
        mu, ls = z[..., :A], z[..., A:].clamp(self.lo, self.hi)
        u = mu + ls.exp() * eps
        return self.scale * torch.tanh(u) + self.bias, squashed_log_prob(u, ls, eps)


class _Critic(torch.nn.Module):
    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, obs=None, action=None):
        x = torch.cat([obs, action], dim=-1)
        for i in range(len(self.net.fc)):
            x = self.net.fc[str(i)](x)
        return self.net.vf_head(x)[..., 0]


def _as_sac(m):
    m = copy.deepcopy(m)
    return _SacActor(m) if hasattr(m, "policy_head") else _Critic(m)


# ------------------------------------------------------------------------ values
def _same(got, want, what):
    """got (value, bar) equals want to 1e-12 of want's largest element, or to a millionth of
    the element's float32 bar where a float64 evaluation itself cancels (the log-std gradient
    at |u| = 40: du sigma eps - d_lp with du sigma eps ~ 80 d_lp)."""
    got, bar = got if isinstance(got, tuple) else (got, 0.0)
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    scale = max(float(np.abs(want).max()) if want.size else 0.0, 1e-300)
    err = np.abs(got - want)
    assert (err <= 1e-12 * scale + 1e-6 * np.asarray(bar)).all(), (what, float(err.max()), scale)


def _flat_grads(grads):
    """[[(dW, db)] per layer] or [dW, db, ...] -> [dW, db, ...]."""
    out = []
    for g in grads:
        if isinstance(g, tuple):
            out += list(g)
        else:
            out.append(g)
    return out


def check_values(case):
    (c, a), (oc, oa) = case.reference(), case.existing()
    assert np.isfinite(c["sums"][0][1]) and np.isfinite(a["sums"][0][1])
    if case.kind == "sac":
        for got, want in zip(c["grads1"] + c["grads2"], oc["critic_grads"] + oc["critic2_grads"]):
            _same(got, want, "critic grads")
        for k in ("q1", "q2", "returns"):
            _same(c[k], oc[k].reshape(-1), k)
        for i in range(2):
            _same(c["sums"][i], oc["sums"][i], f"sums[{i}]")
        for got, want in zip(a["grads"], oa["actor_grads"]):
            _same(got, want, "actor grads")
        _same(a["log_probs"], oa["log_probs"], "log_probs")
        for i in range(2):
            _same(a["sums"][i], oa["sums"][i], f"sums[{i + 2}]")
    elif case.kind == "discrete":
        for got, want in zip(c["grads1"] + c["grads2"], oc["grads1"] + oc["grads2"]):
            _same(got, want, "critic grads")
        for k in ("q1", "q2", "returns"):
            _same(c[k], oc[k], k)
        _same(c["sums"][0], oc["sum_e1"], "sums[0]")
        _same(c["sums"][1], oc["sum_e2"], "sums[1]")
        for got, want in zip(a["grads"], oa["grads"]):
            _same(got, want, "actor grads")
        _same(a["entropies"], oa["entropies"], "entropies")
        _same(a["sums"][0], oa["sum_m"], "sums[2]")
        _same(a["sums"][1], oa["sum_log_pi"], "sums[3]")
    else:
        for got, want in zip(c["grads1"] + c["grads2"], oc["grads"][0] + oc["grads"][1]):
            _same(got, want, "critic grads")
        _same(c["theta"], oc["theta"], "theta")
        _same(c["returns"], oc["returns"], "returns")
        _same(c["q_means"], oc["q_means"], "q_means")
        _same(c["target_means"], oc["target_means"], "target_means")
        _same(c["sums"][0], oc["sum_loss"], "sums[0]")
        _same(c["sums"][1], oc["sum_q"], "sums[1]")
        for got, want in zip(a["grads"], oa["grads"]):
            _same(got, want, "actor grads")
        _same(a["log_probs"], oa["log_probs"], "log_probs")
        _same(a["q_bar"], oa["q_bar"], "q_bar")
        _same(a["sums"][0], oa["sum_q"], "sums[2]")
        _same(a["sums"][1], oa["sum_log_pi"], "sums[3]")
    for ref in (c, a):
        for k, v in ref.items():
            if k == "ok":
                continue
            pairs = v if isinstance(v, list) else [v]
            for p in pairs:
                if isinstance(p, tuple):
                    assert (np.asarray(p[1]) >= 0).all(), k


# (kind, B, n_step, C, E, Np, F, A, actor dims, critic dims, extra)
VALUE_CASES = [
    ("sac", 17, 3, 12, 4, 1, 4, 2, [16, 16], [16, 16], {}),
    ("sac", 40, 2, 9, 4, 3, 3, 1, [], [5], dict(gamma=1.0, done_vals=(0, 1, 2))),
    ("sac", 33, 1, 9, 4, 1, 5, 3, [7], [64, 64], dict(noise_scale=40.0, log_alpha=-10.0,
                                                       log_std_bias=1.0)),
    ("sac", 33, 3, 9, 4, 1, 4, 2, [8], [8], dict(lo=-0.3, hi=0.2, log_alpha=2.0,
                                                 pin=[(0, -0.3), (1, 0.2)])),
    ("discrete", 17, 3, 12, 4, 1, 4, 3, [16, 16], [16], dict(done_vals=(0, 1, 2))),
    ("discrete", 40, 1, 9, 4, 2, 6, 2, [], [], dict(gamma=0.0)),
    ("tqc", 17, 3, 12, 4, 1, 4, 2, [16], [16, 16], dict(N=5, d=2)),
    ("tqc", 30, 2, 9, 4, 1, 3, 1, [], [], dict(N=1, d=0, gamma=1.0)),
    ("tqc", 30, 2, 9, 4, 1, 3, 2, [8], [8], dict(N=8, d=7, ties="exact")),
    ("tqc", 30, 2, 9, 4, 1, 3, 2, [8], [8], dict(N=8, d=3, ties="straddle")),
]


def _case_id(c):
    kind, B, _, _, _, _, F, A, ad, cd, extra = c
    tag = "_".join(f"{k}{v}" for k, v in extra.items() if k in ("N", "d", "ties", "gamma"))
    return f"{kind}_B{B}_F{F}_A{A}_L{len(ad)}{len(cd)}" + (f"_{tag}" if tag else "")


def make_case(c):
    kind, B, n_step, C, E, Np, F, A, ad, cd, extra = c
    return Case(kind, B, n_step, C, E, Np, F, A, ad, cd, **extra)


@pytest.mark.parametrize("c", VALUE_CASES, ids=[_case_id(c) for c in VALUE_CASES])
def test_values_match_the_existing_references(c):
    check_values(make_case(c))


def test_discrete_log_softmax_keeps_underflowing_probabilities():
    """Logit gaps of 40 and 100: pi underflows float32 (exp(-100)) but log pi stays finite and
    its bar small; the value is the log-softmax, never the log of a softmax."""
    for gap in (40.0, 100.0):
        z = np.array([[gap, 0.0, -1.0], [0.0, gap, 3.0]], np.float32).astype(np.float64)
        lp, pi = sb.log_softmax((z, np.zeros_like(z)))
        want = dsref.log_softmax(z)
        assert np.abs(lp[0] - want).max() <= 1e-12 * gap
        assert (lp[1] <= 1e-5 * (np.abs(lp[0]) + 1)).all()
        assert (pi[0] >= 0).all() and (pi[1] < 1e-6).all()


def test_the_primitives_bound_their_float32_evaluations():
    """tanhf, log1pf, softplus (both sides of 20) and squashed_dim against a float32 evaluation
    whose every operation is correctly rounded, on a sweep of inputs with |u| up to 40; and each
    bar holds the claimed ulps of its result."""
    f32 = lambda t: np.float32(t).astype(np.float64)  # noqa: E731
    g = np.random.default_rng(0)
    x = f32(np.concatenate([g.uniform(-40, 40, 4000), np.linspace(-21, 21, 4001)]))
    zero = np.zeros_like(x)
    ulp = lambda t: np.spacing(np.abs(np.float32(t))).astype(np.float64)  # noqa: E731
    v, b = sb.f_tanh((x, zero))
    assert (np.abs(f32(np.tanh(x)) - v) <= b).all() and (b >= 2 * ulp(v) * 0.99).all()
    v, b = sb.f_log1p((np.abs(x), zero))
    assert (np.abs(f32(np.log1p(np.abs(x))) - v) <= b).all() and (b >= ulp(v) * 0.99).all()
    v, b = sb.f_softplus((x, zero))
    sp = np.where(x > 20, x, f32(np.log1p(f32(np.exp(x)))))
    assert (np.abs(sp - v) <= b).all()
    mu = f32(g.standard_normal((500, 3)))
    raw = f32(g.uniform(-4, 3, (500, 3)))
    eps = f32(20 * g.standard_normal((500, 3)))
    s = sb.squashed_dim((mu, np.zeros((500, 3))), (raw, np.zeros((500, 3))), eps, -2.0, 1.0)
    ls = np.clip(raw, -2.0, 1.0)
    u = f32(f32(np.exp(ls)) * eps + mu)
    xx = -2.0 * u
    sp = np.where(xx > 20, xx, f32(np.log1p(f32(np.exp(xx)))))
    corr = 2.0 * f32(f32(f32(np.log(2.0)) - u) - sp)
    term = f32(f32(f32(f32(-0.5 * eps * eps) - ls) - f32(0.5 * np.log(2 * np.pi))) - corr)
    for got, key in ((u, "u"), (f32(np.tanh(u)), "y"), (term, "term")):
        assert (np.abs(got - s[key][0]) <= s[key][1]).all(), key
    assert (s["ls"][1] == 0).all()


# ------------------------------------------------------------------------ soundness
def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


def _torch_sac(case):
    """Float32 autograd through algorithms/sac.py's sampled losses on the case's windows."""
    from warp_drive_b200.training.algorithms.sac import (SAC, torch_actor_loss,
                                                         torch_sampled_critic_loss)

    actor, c1, c2, t1, t2 = (_as_sac(m) for m in case.models)
    algo = SAC(discount_factor_gamma=case.gamma, n_step=case.n_step, action_dim=case.A)
    la = torch.tensor([case.log_alpha], dtype=torch.float32)
    obs, act, rew, done, boot = (_t(x).float() for x in case.rows())
    l1, l2, q1, q2, R = torch_sampled_critic_loss(algo, actor, t1, t2, c1, c2, la, obs, act, rew,
                                                  done, boot, _t(case.noise_c))
    g1 = torch.autograd.grad(l1 + l2, list(c1.parameters()) + list(c2.parameters()))
    loss, q, lp = torch_actor_loss(algo, actor, c1, c2, la, obs, _t(case.noise_a))
    ga = torch.autograd.grad(loss, list(actor.parameters()))
    n = len(g1) // 2
    return ({"grads1": g1[:n], "grads2": g1[n:], "q1": q1, "q2": q2, "returns": R},
            {"grads": ga, "log_probs": lp})


def _torch_discrete(case):
    from warp_drive_b200.training.algorithms.sac_discrete import DiscreteSAC

    actor, c1, c2, t1, t2 = case.models
    algo = DiscreteSAC(discount_factor_gamma=case.gamma, n_step=case.n_step, n_actions=case.A)
    alpha = torch.tensor(case.log_alpha, dtype=torch.float32).exp()
    obs, act, rew, done, boot = case.rows()
    obs, boot, rew = _t(obs).float(), _t(boot).float(), _t(rew).float()
    done = _t(done.astype(np.float32))

    def run(net, x):
        for i in range(len(net.fc)):
            x = net.fc[str(i)](x)
        return (net.policy_head if hasattr(net, "policy_head") else net.vf_head)(x)

    with torch.no_grad():
        log_pi = torch.log_softmax(run(actor, boot), -1)
        m = torch.minimum(run(t1, boot), run(t2, boot))
        R = algo.sampled_returns(rew, done, (log_pi.exp() * (m - alpha * log_pi)).sum(-1))
    a = torch.from_numpy(np.asarray(act, np.int64)).reshape(-1, 1)
    q1, q2 = run(c1, obs).gather(-1, a)[..., 0], run(c2, obs).gather(-1, a)[..., 0]
    l1, l2 = algo.critic_losses(q1, q2, R)
    g = torch.autograd.grad(l1 + l2, list(c1.parameters()) + list(c2.parameters()))
    log_pi = torch.log_softmax(run(actor, obs), -1)
    with torch.no_grad():
        m = torch.minimum(run(c1, obs), run(c2, obs))
    loss = (log_pi.exp() * (alpha * log_pi - m)).sum(-1).mean()
    ga = torch.autograd.grad(loss, list(actor.parameters()))
    n = len(g) // 2
    return ({"grads1": g[:n], "grads2": g[n:], "q1": q1, "q2": q2, "returns": R},
            {"grads": ga, "entropies": -(log_pi.exp() * log_pi).sum(-1)})


def _torch_tqc(case):
    from warp_drive_b200.training.algorithms.tqc import TQC

    actor, c1, c2, t1, t2 = case.models
    sa = _SacActor(actor)
    algo = TQC(discount_factor_gamma=case.gamma, n_step=case.n_step, action_dim=case.A,
               n_critics=2, n_quantiles=case.N, drop_per_net=case.d)
    alpha = torch.tensor(case.log_alpha, dtype=torch.float32).exp()
    obs, act, rew, done, boot = (_t(x).float() for x in case.rows())

    def q(net, o, a):
        x = torch.cat([o, a], -1)
        for i in range(len(net.fc)):
            x = net.fc[str(i)](x)
        return net.vf_head(x)

    with torch.no_grad():
        a_t, lp_t = sa.sample(boot, _t(case.noise_c))
        atoms = torch.stack([q(t1, boot, a_t), q(t2, boot, a_t)], 1)
        T = algo.truncated_returns(rew, done, atoms, lp_t, alpha)
    theta = torch.stack([q(c1, obs, act), q(c2, obs, act)], 1)
    loss = algo.quantile_huber_loss(theta, T)
    g = torch.autograd.grad(loss, list(c1.parameters()) + list(c2.parameters()))
    a, lp = sa.sample(obs, _t(case.noise_a))
    qbar = torch.stack([q(c1, obs, a), q(c2, obs, a)], 1).mean(dim=(-2, -1))
    ga = torch.autograd.grad((alpha * lp - qbar).mean(), list(sa.parameters()))
    n = len(g) // 2
    return ({"grads1": g[:n], "grads2": g[n:], "returns": T}, {"grads": ga, "log_probs": lp})


SOUND_CASES = [
    ("sac", 97, 3, 12, 4, 1, 4, 2, [16, 16], [16, 16], {}),
    ("sac", 65, 2, 9, 4, 1, 3, 1, [8], [8], dict(lo=-0.3, hi=0.2, noise_scale=8.0)),
    ("discrete", 97, 3, 12, 4, 1, 4, 3, [16, 16], [16, 16], dict(done_vals=(0, 1, 2))),
    ("discrete", 65, 2, 9, 4, 1, 5, 4, [8], [], {}),
    ("tqc", 97, 3, 12, 4, 1, 4, 2, [16], [16, 16], dict(N=5, d=2)),
    ("tqc", 65, 2, 9, 4, 1, 3, 1, [8], [8], dict(N=8, d=3, ties="straddle")),
]


@pytest.mark.parametrize("c", SOUND_CASES, ids=[_case_id(c) for c in SOUND_CASES])
def test_a_float32_torch_update_lies_within_the_bars(c):
    case = make_case(c)
    ref_c, ref_a = case.reference()
    got_c, got_a = {"sac": _torch_sac, "discrete": _torch_discrete, "tqc": _torch_tqc}[
        case.kind](case)
    for k in ("grads1", "grads2"):
        for i, (g, want) in enumerate(zip(got_c[k], ref_c[k])):
            within(g.double().numpy(), want, f"{k}[{i}]")
    for i, (g, want) in enumerate(zip(got_a["grads"], ref_a["grads"])):
        within(g.double().numpy(), want, f"actor grads[{i}]")
    for k in ("q1", "q2", "returns"):
        if k in got_c:
            within(got_c[k].detach().double().numpy(), ref_c[k], k)
    for k in ("log_probs", "entropies"):
        if k in got_a:
            within(got_a[k].detach().double().numpy(), ref_a[k], k)


# ------------------------------------------------------------------------ sensitivity
def _norm_ok(got, value):
    return float(np.linalg.norm(got - value) / max(np.linalg.norm(value), 1e-30)) <= 2e-4


def _bars_ok(got, ref):
    v, b = ref
    return bool((np.abs(got - v) <= b).all())


def _zero_small(ref):
    """Zero the smallest elements, as far as the norm-wise check still accepts."""
    v = ref[0]
    got, zeroed = v.copy(), 0
    for i in np.argsort(np.abs(v), axis=None):
        trial = got.copy()
        trial.flat[i] = 0.0
        if not _norm_ok(trial, v) or v.flat[i] == 0.0:
            if v.flat[i] == 0.0:
                continue
            break
        got, zeroed = trial, zeroed + 1
    return got, zeroed


def test_per_element_bars_reject_defects_the_norm_wise_check_accepts():
    # ---- SAC: zero the small elements of the actor's second-layer gradient, scale the critic's
    sac = make_case(("sac", 333, 3, 40, 6, 1, 4, 2, [64, 64], [64, 64], {}))
    ref_c, ref_a = sac.reference()
    g = ref_a["grads"][2]
    got, zeroed = _zero_small(g)
    assert zeroed > 10 and _norm_ok(got, g[0]) and not _bars_ok(got, g)
    g = ref_c["grads1"][2]
    got = g[0] * (1 + 1e-4)
    assert _norm_ok(got, g[0]) and not _bars_ok(got, g)
    got = g[0].copy()                                   # gross: a whole row dropped
    got[np.argmax(np.abs(g[0]).sum(axis=1))] = 0.0
    assert not _norm_ok(got, g[0]) and not _bars_ok(got, g)

    # ---- discrete SAC: flip the sign of the smallest logit deltas
    dsc = make_case(("discrete", 2113, 3, 40, 16, 1, 4, 3, [64, 64], [64, 64], {}))
    ref_a = dsc.reference()[1]
    delta = ref_a["logit_deltas"]
    v = delta[0]
    got, flipped = v.copy(), 0                          # smallest first, while the norm accepts
    for i in np.argsort(np.abs(v), axis=None):
        if abs(v.flat[i]) <= delta[1].flat[i]:
            continue
        trial = got.copy()
        trial.flat[i] = -trial.flat[i]
        if not _norm_ok(trial, v):
            break
        got, flipped = trial, flipped + 1
    assert flipped >= 3 and _norm_ok(got, v) and not _bars_ok(got, delta)
    got = v.copy()                                      # gross: action 0's deltas flipped
    got[:, 0] = -got[:, 0]
    assert not _norm_ok(got, v) and not _bars_ok(got, delta)
    # (the actor's gradient bars carry h - sum pi h's cancellation: wider than 1e-4 of it)
    ga = dsc.reference()[0]["grads1"][2]
    got = ga[0] * (1 + 1e-4)
    assert _norm_ok(got, ga[0]) and not _bars_ok(got, ga)

    # ---- TQC: one row of a 2113-row batch reads another row's kept atom (a stale tile slot)
    tqc = make_case(("tqc", 2113, 3, 40, 16, 1, 4, 2, [16], [16, 16], dict(N=5, d=2)))
    ref_c = tqc.reference()[0]
    T, tm = ref_c["returns"], ref_c["target_means"]
    K = T[0].shape[1]
    # the donor: the other row whose atom 3 lies closest to row 1000's (a plausible stale value)
    diff = np.abs(T[0][:, 3] - T[0][1000, 3])
    diff[1000] = np.inf
    donor = int(np.argmin(np.where(diff > 0, diff, np.inf)))
    got = tm[0].copy()
    got[1000] += (T[0][donor, 3] - T[0][1000, 3]) / K
    assert _norm_ok(got, tm[0]) and not _bars_ok(got, tm)
    got = T[0].copy()
    got[1000, 3] = T[0][donor, 3]
    assert _norm_ok(got, T[0]) and not _bars_ok(got, T)
    got = tm[0] + (np.roll(T[0][:, 3], 1) - T[0][:, 3]) / K   # gross: every row's atom 3 stale
    assert not _norm_ok(got, tm[0]) and not _bars_ok(got, tm)
