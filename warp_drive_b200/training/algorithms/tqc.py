"""TQC (Kuznetsov et al., "Controlling Overestimation Bias with Truncated Mixture of Continuous
Distributional Quantile Critics", 2020) on the replay buffer's sampled n-step windows: SAC's
tanh-squashed Gaussian actor and temperature, M distributional critics of N quantiles each
(`fully_connected_quantile_critic`, held together by QuantileCritics) with their targets, and a
bootstrap truncated to the K = M (N - d) smallest of the M N pooled target atoms.  There is no
target actor.

The torch statement of wdb_tqc_{critic,actor}_update_sampled (include/wdb200.h), which TrainerTQC
runs for the shapes the native passes do not take (any M, N, d); tests/tqc_reference.py restates
both passes in float64 NumPy.  Per sampled window g, with fresh standard normals eps' (critic) and
eps (actor) per update and tau_i = (2i + 1) / (2N) in float32:
    a', log pi' = the actor's sample at obs'
    y_0 <= .. <= y_{K-1} = the K smallest target atoms Z'_m,j(obs', a'), pooled at index m N + j
                           (a stable sort: ties to the lower index)
    T_k  = SAC's n-step return bootstrapped with y_k - alpha log pi'
    critic loss = mean over (g, m, i, k) of |tau_i - 1{u < 0}| H(u),  u = T_k - theta_m,i(obs, a),
                  H the Huber function with kappa = 1            (reaches only the critics)
    a, log pi = the actor's sample at obs
    actor loss  = mean over g of (alpha log pi - mean over (m, i) of theta_m,i(obs, a))
                                                                 (reaches only the actor)
    d loss / d log_alpha = SAC's.
"""
import torch

from warp_drive_b200.training.algorithms.sac import SAC


class TQC(SAC):
    """SAC's temperature, alpha gradient and actor metrics with M quantile critics of N quantiles
    each and `drop_per_net` top quantiles dropped per critic from the pooled bootstrap."""

    def __init__(self, discount_factor_gamma=1.0, normalize_advantage=False,
                 normalize_return=False, n_step=1, alpha=0.2, autotune_alpha=True,
                 target_entropy=None, action_dim=1, n_critics=2, n_quantiles=25,
                 drop_per_net=2):
        integer = lambda v: isinstance(v, int) and not isinstance(v, bool)  # noqa: E731
        if not integer(n_critics) or n_critics < 1:
            raise ValueError(f"n_critics must be an integer >= 1, got {n_critics!r}")
        if not integer(n_quantiles) or not 2 <= n_quantiles <= 64:
            raise ValueError(f"num_quantiles must be an integer in [2, 64], got {n_quantiles!r}")
        if not integer(drop_per_net) or not 0 <= drop_per_net < n_quantiles:
            raise ValueError(f"top_quantiles_to_drop_per_net must be an integer in [0, "
                             f"{n_quantiles - 1}], got {drop_per_net!r}")
        super().__init__(discount_factor_gamma, normalize_advantage, normalize_return, n_step,
                         alpha=alpha, autotune_alpha=autotune_alpha,
                         target_entropy=target_entropy, action_dim=action_dim)
        self.n_critics = n_critics
        self.n_quantiles = n_quantiles
        self.drop_per_net = drop_per_net

    @property
    def kept_atoms(self):
        """K: the pooled target atoms the bootstrap keeps."""
        return self.n_critics * (self.n_quantiles - self.drop_per_net)

    def quantile_fractions(self, dtype=torch.float32, device=None):
        """tau_i = (2i + 1) / (2N), i = 0 .. N - 1, rounded once to float32."""
        N = self.n_quantiles
        tau = torch.tensor([(2 * i + 1) / (2 * N) for i in range(N)], dtype=torch.float32)
        return tau.to(dtype=dtype, device=device)

    def truncated_returns(self, rewards, done, atoms, log_pi, alpha):
        """T [B, K]: SAC's n-step return of each kept atom.  rewards and done [n_step, B], the
        target atoms [B, M, N], log pi' [B], alpha a tensor [1]."""
        pooled = atoms.reshape(atoms.shape[0], -1)
        kept = torch.sort(pooled, dim=-1, stable=True).values[:, :self.kept_atoms]
        boot = kept - alpha * log_pi[:, None]
        return self.sampled_returns(rewards[..., None], done[..., None], boot)

    def quantile_huber_loss(self, theta, returns):
        """The mean over (g, m, i, k) of |tau_i - 1{u < 0}| H(u), u = T_k - theta_m,i: theta
        [B, M, N], returns [B, K]."""
        u = returns[:, None, None, :] - theta[..., None]
        tau = self.quantile_fractions(theta.dtype, theta.device)[:, None]
        au = u.abs()
        huber = torch.where(au <= 1.0, 0.5 * u * u, au - 0.5)
        return ((tau - (u < 0).to(u.dtype)).abs() * huber).mean()

    @staticmethod
    def critic_metrics(critic_loss, mean_q, mean_return):
        """The logged critic metrics of one update, as floats: the loss, the mean quantile of
        the critics at (obs, a) and the mean of the kept atoms' returns."""
        return {"Critic loss": float(critic_loss), "Mean Q value": float(mean_q),
                "Mean return": float(mean_return)}


def torch_sampled_critic_loss(algo, actor, target_critics, critics, log_alpha, obs, actions,
                              rewards, done, boot_obs, noise):
    """The critic loss over B sampled windows gathered from the replay buffer: obs and boot_obs
    [B, F], actions [B, A], rewards and done [n_step, B], noise [B, A] (eps'); target_critics and
    critics QuantileCritics.  Returns (loss, theta [B, M, N], returns [B, K]); only the critics
    take gradients."""
    with torch.no_grad():
        a_t, log_pi = actor.sample(boot_obs, noise)
        returns = algo.truncated_returns(rewards, done, target_critics(obs=boot_obs, action=a_t),
                                         log_pi, log_alpha.exp())
    theta = critics(obs=obs, action=actions)
    return algo.quantile_huber_loss(theta, returns), theta, returns


def torch_actor_loss(algo, actor, critics, log_alpha, obs_rows, noise):
    """mean(alpha log pi - mean_m,i theta_m,i(obs, a)) over obs_rows [B, F] with eps = noise
    [B, A]; returns (loss, Qbar [B], log pi [B]).  Call .backward(inputs=actor parameters) to
    keep the critics' and log_alpha's gradients out."""
    a, log_pi = actor.sample(obs_rows, noise)
    q = critics(obs=obs_rows, action=a).mean(dim=(-2, -1))
    loss = (log_alpha.detach().exp() * log_pi - q).mean()
    return loss, q, log_pi
