"""DQN objective over sampled n-step windows: double DQN (van Hasselt et al. 2016) with n-step
returns and a Huber loss (Mnih et al. 2015).

The torch statement of wdb_dqn_update_sampled (include/wdb200.h): TrainerDQN runs it for the
shapes the native pass does not take, and tests/dqn_update_reference.py restates it in float64
NumPy.  QuantileDQN is quantile-regression DQN on the same windows (wdb_qr_dqn_update_sampled,
tests/qr_dqn_reference.py), ImplicitQuantileDQN implicit quantile networks
(wdb_iqn_update_sampled, tests/iqn_reference.py), CategoricalDQN categorical DQN
(wdb_c51_update_sampled, tests/c51_reference.py), BranchingDQN action branching over the heads of
a MultiDiscrete space (wdb_branching_dqn_update_sampled, tests/branching_q_reference.py).

Action masks: every loss takes `boot_mask` [B, A], obs' own action mask; the bootstrap's argmax /
max then ranges over its valid actions (masked_scores), the rule of wdb_dqn_update_masked and
wdb_c51_update_masked.  None gives the unmasked ops."""
import torch
from torch.nn import functional as func


def masked_scores(scores, boot_mask):
    """scores [B, A] with the actions boot_mask [B, A] marks invalid (zero) at -inf, for the
    bootstrap's argmax / max over obs' valid actions; a row with no valid action keeps every
    action (the unmasked rule).  boot_mask None: scores itself."""
    if boot_mask is None:
        return scores
    valid = boot_mask != 0
    valid = valid | ~valid.any(dim=-1, keepdim=True)
    return scores.masked_fill(~valid, float("-inf"))


class DQN:
    # TrainerDQN runs this policy's update as native kernels (fused_dqn.py) when the shapes
    # allow it; False keeps the torch autograd update below (a test switch, not a config key)
    use_fused_update = True

    def __init__(self, discount_factor_gamma=1.0, n_step=1, double_q=True, huber_delta=1.0):
        assert 0 <= discount_factor_gamma <= 1
        assert n_step >= 1
        if not huber_delta > 0:
            raise ValueError(f"huber_delta must be > 0, got {huber_delta}")
        self.discount_factor_gamma = discount_factor_gamma
        self.n_step = n_step
        self.double_q = bool(double_q)
        self.huber_delta = float(huber_delta)
        self.normalize_return = False

    def sampled_returns(self, rewards, done, boot):
        """The n-step returns [B] of B sampled windows: rewards and done flags [n_step, B] of
        each window's steps and its bootstrap value `boot` [B]:
        R = r_0 + m_0 gamma (r_1 + ... m_{n-1} gamma boot) with m_j = (done_j == 0), so every
        non-zero flag (MountainCar's 2 at the goal included) ends the window; the operation
        order of DDPG.sampled_returns and of the native pass."""
        live = (done == 0).to(rewards.dtype)
        r = boot
        for j in reversed(range(self.n_step)):
            r = live[j] * self.discount_factor_gamma * r + rewards[j]
        return r

    def bootstrap(self, q_net, target_net, boot_obs, boot_mask=None):
        """The bootstrap value [B] at the windows' last observation (no gradient):
        target(obs')[argmax online(obs')] with double_q (the first maximum), else
        max target(obs').  boot_mask [B, A]: obs' own action mask; the argmax / max range over
        its valid actions (masked_scores)."""
        with torch.no_grad():
            q_target = target_net.q_values(boot_obs)
            if self.double_q:
                best = masked_scores(q_net.q_values(boot_obs), boot_mask).argmax(
                    dim=-1, keepdim=True)
                return q_target.gather(-1, best)[..., 0]
            return masked_scores(q_target, boot_mask).max(dim=-1).values

    def loss(self, q_net, target_net, obs, actions, rewards, done, boot_obs, weights=None,
             boot_mask=None):
        """(Huber loss, Q(obs, a) [B], R [B]) of B sampled windows: obs [B, F], actions [B, 1]
        (int), rewards / done [n_step, B], boot_obs [B, F].  weights [B]: prioritized replay's
        importance-sampling weights, the loss (1/B) sum w_g huber(Q_g - R_g) of
        wdb_dqn_update_prioritized.  boot_mask [B, A]: obs' action mask (wdb_dqn_update_masked)."""
        with torch.no_grad():
            returns = self.sampled_returns(rewards, done, self.bootstrap(
                q_net, target_net, boot_obs, boot_mask))
        q = q_net.q_values(obs).gather(-1, actions.long().reshape(-1, 1))[..., 0]
        if weights is None:
            loss = func.huber_loss(q, returns, delta=self.huber_delta)
        else:
            loss = (weights * func.huber_loss(q, returns, reduction="none",
                                              delta=self.huber_delta)).mean()
        return loss, q, returns

    @staticmethod
    def loss_metrics(loss, mean_q, returns):
        """The logged metrics of one update: the loss and the mean Q(obs, a) as floats, the mean
        of the returns [B]."""
        return {"Q loss": float(loss), "Mean Q value": float(mean_q),
                "Mean return": float(returns.double().mean())}


class BranchingDQN(DQN):
    """Branching DQN (Tavakoli, Pardo & Kormushev 2018) on DQN's windows and n-step recursion,
    for a FullyConnectedBranchingQ: the torch statement of wdb_branching_dqn_update_sampled
    (include/wdb200.h), restated in float64 NumPy by tests/branching_q_reference.py.  Heads
    d = 0 .. D-1 are column blocks of the one Q head; each head bootstraps as DQN does and the
    return is built on their mean (BDQ's mean target), shared by every head's loss."""

    def bootstrap(self, q_net, target_net, boot_obs, boot_mask=None):
        """(1/D) sum_d boot_d [B] (no gradient), boot_d = target_d(obs')[argmax online_d(obs')]
        with double_q (the first maximum), else max target_d(obs'); summed in ascending d."""
        assert boot_mask is None, "branching DQN takes no action mask"
        with torch.no_grad():
            targets = q_net.branches(target_net.q_values(boot_obs))
            online = q_net.branches(q_net.q_values(boot_obs)) if self.double_q else targets
            total = None
            for qt, qc in zip(targets, online):
                b = qt.gather(-1, qc.argmax(dim=-1, keepdim=True))[..., 0]
                total = b if total is None else total + b
            return total / len(targets)

    def loss(self, q_net, target_net, obs, actions, rewards, done, boot_obs, weights=None,
             boot_mask=None):
        """(loss, Q-bar [B], R [B]) of B sampled windows, the arguments of DQN.loss with actions
        [B, D]: (1/B) sum_g w_g (1/D) sum_d huber(Q_d(obs, a_d) - R_g, delta), w = 1 without
        weights, and Q-bar = (1/D) sum_d Q_d(obs, a_d), which feeds the metrics and the
        priorities."""
        with torch.no_grad():
            returns = self.sampled_returns(rewards, done, self.bootstrap(
                q_net, target_net, boot_obs, boot_mask))
        heads = q_net.branches(q_net.q_values(obs))
        a = actions.long().reshape(obs.shape[0], len(heads))
        q = torch.stack([h.gather(-1, a[:, d:d + 1])[..., 0] for d, h in enumerate(heads)], -1)
        rows = func.huber_loss(q, returns[:, None].expand_as(q), reduction="none",
                               delta=self.huber_delta).mean(dim=-1)
        loss = rows.mean() if weights is None else (weights * rows).mean()
        return loss, q.mean(dim=-1), returns


class QuantileDQN(DQN):
    """Quantile-regression DQN (Dabney et al. 2018) on DQN's windows, n-step recursion and
    bootstrap rule: the torch statement of wdb_qr_dqn_update_sampled (include/wdb200.h) for a
    FullyConnectedQuantileQ, restated in float64 NumPy by tests/qr_dqn_reference.py.
    `huber_delta` is the quantile Huber loss's kappa."""

    def bootstrap_quantiles(self, q_net, target_net, boot_obs, boot_mask=None):
        """target(obs')[a*] [B, N] (no gradient), a* the first argmax of the mean quantile of
        online(obs') with double_q, else of target(obs'); over obs' valid actions with
        boot_mask [B, A]."""
        with torch.no_grad():
            boot = target_net.quantiles(boot_obs)
            chooser = q_net.quantiles(boot_obs) if self.double_q else boot
            best = masked_scores(chooser.mean(dim=-1), boot_mask).argmax(dim=-1)
            return boot[torch.arange(boot.shape[0], device=boot.device), best]

    def loss(self, q_net, target_net, obs, actions, rewards, done, boot_obs, weights=None,
             boot_mask=None):
        """(quantile Huber loss, Q-bar [B], R-bar [B]) of B sampled windows, the arguments of
        DQN.loss.  theta_i = quantiles(obs)[a, i] at tau_i = (2i + 1) / (2N), T_j the n-step
        recursion on each bootstrap quantile, u_ij = T_j - theta_i, and the row loss
        (1/N) sum_i sum_j |tau_i - 1{u_ij < 0}| huber(u_ij, kappa) / kappa; the loss is the mean
        over rows of w_g times it (w = 1 without weights).  Q-bar = mean_i theta_i and
        R-bar = mean_j T_j feed the metrics and the priorities."""
        with torch.no_grad():
            boot = self.bootstrap_quantiles(q_net, target_net, boot_obs, boot_mask)
            targets = self.sampled_returns(rewards[..., None], done[..., None], boot)
        quantiles = q_net.quantiles(obs)
        n = quantiles.shape[-1]
        theta = quantiles[torch.arange(quantiles.shape[0], device=quantiles.device),
                          actions.long().reshape(-1)]
        tau = (2 * torch.arange(n, device=theta.device, dtype=theta.dtype) + 1) / (2 * n)
        u = targets[:, None, :] - theta[:, :, None]             # [B, i, j]
        below = (u.detach() < 0).to(theta.dtype)
        rho = (tau[:, None] - below).abs() * func.huber_loss(
            u, torch.zeros_like(u), reduction="none", delta=self.huber_delta) / self.huber_delta
        rows = rho.sum(dim=1).mean(dim=-1)
        loss = rows.mean() if weights is None else (weights * rows).mean()
        return loss, theta.mean(dim=-1), targets.mean(dim=-1)


class ImplicitQuantileDQN(DQN):
    """Implicit quantile networks (IQN; Dabney, Ostrovski, Silver & Munos 2018) on DQN's
    windows, n-step recursion and bootstrap rule: the torch statement of wdb_iqn_update_sampled
    (include/wdb200.h) for a FullyConnectedIQN, restated in float64 NumPy by
    tests/iqn_reference.py.  The levels come in: `taus` [B, N + N'] holds each loss row's N
    online levels tau_i, then its N' target levels tau'_j.  `huber_delta` is kappa."""

    def bootstrap_quantiles(self, q_net, target_net, boot_obs, taus_prime, boot_mask=None):
        """The target's Z at tau'_j of a* [B, N'] (no gradient), a* the first argmax of the
        collapsed Q of online(obs') with double_q, else of target(obs'); over obs' valid
        actions with boot_mask [B, A]."""
        with torch.no_grad():
            best = masked_scores((q_net if self.double_q else target_net).q_values(boot_obs),
                                 boot_mask).argmax(dim=-1)
            z = target_net.quantiles_at(boot_obs, taus_prime)           # [B, N', A]
            return z.gather(-1, best[:, None, None].expand(-1, z.shape[1], 1))[..., 0]

    def loss(self, q_net, target_net, obs, actions, rewards, done, boot_obs, weights=None,
             taus=None, boot_mask=None):
        """(quantile Huber loss, Q-bar [B], R-bar [B]) of B sampled windows, the arguments of
        DQN.loss and the levels `taus`.  theta_i = Z_tau_i(obs)[a], T_j the n-step recursion on
        the target's Z_tau'_j(obs')[a*], u_ij = T_j - theta_i, and the row loss
        (1/N') sum_i sum_j |tau_i - 1{u_ij < 0}| huber(u_ij, kappa) / kappa; the loss is the mean
        over rows of w_g times it (w = 1 without weights).  Q-bar = mean_i theta_i and
        R-bar = mean_j T_j feed the metrics and the priorities."""
        n = q_net.num_tau_samples
        assert taus is not None and taus.shape == (obs.shape[0], n + q_net.num_tau_prime_samples)
        tau, tau_prime = taus[:, :n].to(obs.dtype), taus[:, n:].to(obs.dtype)
        with torch.no_grad():
            boot = self.bootstrap_quantiles(q_net, target_net, boot_obs, tau_prime, boot_mask)
            targets = self.sampled_returns(rewards[..., None], done[..., None], boot)
        z = q_net.quantiles_at(obs, tau)                                 # [B, N, A]
        a = actions.long().reshape(-1)
        theta = z.gather(-1, a[:, None, None].expand(-1, n, 1))[..., 0]  # [B, N]
        u = targets[:, None, :] - theta[:, :, None]                      # [B, i, j]
        below = (u.detach() < 0).to(theta.dtype)
        rho = (tau[:, :, None] - below).abs() * func.huber_loss(
            u, torch.zeros_like(u), reduction="none", delta=self.huber_delta) / self.huber_delta
        rows = rho.sum(dim=1).mean(dim=-1)
        loss = rows.mean() if weights is None else (weights * rows).mean()
        return loss, theta.mean(dim=-1), targets.mean(dim=-1)


class CategoricalDQN(DQN):
    """Categorical DQN (C51; Bellemare, Dabney & Munos 2017) on DQN's windows, n-step recursion
    and bootstrap rule: the torch statement of wdb_c51_update_sampled (include/wdb200.h) for a
    FullyConnectedCategoricalQ, restated in float64 NumPy by tests/c51_reference.py.  C51 has no
    Huber loss: `huber_delta` is not used (TrainerDQN refuses it in a categorical policy's
    config).

    Priorities: prioritized replay writes (|Q-bar - R-bar| + epsilon)^alpha, as for QR-DQN and
    IQN, so the store is shared by every Q network; Rainbow uses the row's cross-entropy
    instead -- a deliberate divergence."""

    def bootstrap_distribution(self, q_net, target_net, boot_obs, boot_mask=None):
        """p' = softmax(target.logits(obs')[a*]) [B, N] (no gradient), a* the first argmax of
        the expectation of online(obs') with double_q, else of target(obs'); over obs' valid
        actions with boot_mask [B, A] (wdb_c51_update_masked)."""
        with torch.no_grad():
            best = masked_scores((q_net if self.double_q else target_net).q_values(boot_obs),
                                 boot_mask).argmax(dim=-1)
            p = target_net.probabilities(boot_obs)
            return p[torch.arange(p.shape[0], device=p.device), best]

    def loss(self, q_net, target_net, obs, actions, rewards, done, boot_obs, weights=None,
             boot_mask=None):
        """(cross-entropy loss, Q-bar [B], R-bar [B]) of B sampled windows, the arguments of
        DQN.loss.  Tz_j is the n-step recursion on each atom z_j, clamped to [z_0, z_{N-1}];
        the projection m_i = sum_j clip(1 - |Tz_j - z_i| / dz, 0, 1) p'_j (Dopamine's dense
        form); the row loss -sum_i m_i log_softmax(l)_i over the online logits l of the row's
        action, and the loss the mean over rows of w_g times it (w = 1 without weights).
        Q-bar = sum_i z_i p_i and R-bar = sum_i z_i m_i feed the metrics and the priorities."""
        z = q_net.support.to(obs.dtype)
        with torch.no_grad():
            p_boot = self.bootstrap_distribution(q_net, target_net, boot_obs, boot_mask)
            tz = self.sampled_returns(rewards[..., None], done[..., None],
                                      z.expand(obs.shape[0], -1))
            tz = tz.clamp(z[0], z[-1])
            pair = (1 - (tz[:, None, :] - z[None, :, None]).abs() / q_net.delta_z).clamp(0, 1)
            m = (pair * p_boot[:, None, :]).sum(dim=-1)                 # [B, i]
        logits = q_net.logits(obs)
        logits = logits[torch.arange(logits.shape[0], device=logits.device),
                        actions.long().reshape(-1)]                      # [B, N]
        rows = -(m * func.log_softmax(logits, dim=-1)).sum(dim=-1)
        loss = rows.mean() if weights is None else (weights * rows).mean()
        qbar = (torch.softmax(logits.detach(), dim=-1) * z).sum(dim=-1)
        return loss, qbar, (m * z).sum(dim=-1)
