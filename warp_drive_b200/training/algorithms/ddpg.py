"""DDPG objective: n-step bootstrapped critic target + deterministic policy gradient
(warp_drive/training/algorithms/policygradient/ddpg.py:17-177).

Same mathematics, including the reference's treatment of the LAST timestep of the batch
(bootstrapped with the final next-value WITHOUT discount and without its reward unless the
episode ended there, ddpg.py:68-73); the n-step recursion runs as `n_step` whole-batch tensor
expressions instead of the reference's `valid_range x n_step` Python double loop of tiny
launches (results identical: tests/test_ddpg_cpu.py compares against vectors produced by the
reference class itself)."""
import torch
from torch import nn

_EPSILON = 1e-10


class DDPG:
    # TrainerDDPG runs this policy's update as native kernels (fused_ddpg.py) when the shapes
    # allow it; False keeps the torch autograd update below (a test switch, not a config key)
    use_fused_update = True

    def __init__(self, discount_factor_gamma=1.0, normalize_advantage=False,
                 normalize_return=False, n_step=1):
        assert 0 <= discount_factor_gamma <= 1
        assert n_step >= 1
        self.discount_factor_gamma = discount_factor_gamma
        self.normalize_advantage = normalize_advantage
        self.normalize_return = normalize_return
        self.n_step = n_step

    @staticmethod
    def _normalize(x):
        return (x - x.mean(dim=(1, 2), keepdim=True)) / (x.std(dim=(1, 2), keepdim=True) + _EPSILON)

    def n_step_returns(self, rewards, done_flags, next_values):
        """rewards [T, E, Np], done_flags [T, E] (0/1), next_values [T-1, E, Np] (detached)
        -> returns [T - n_step + 1, E, Np]  (ddpg.py:62-79)."""
        return self.window_returns(rewards, done_flags, next_values[self.n_step - 1:],
                                   next_values[-1])

    def window_returns(self, rewards, done_flags, boot, boot_last):
        """The n-step returns [T - n_step + 1, E, Np] from each window's bootstrap value:
        `boot` [T - n_step, E, Np] for the windows whose last step has a successor inside the
        batch, `boot_last` [E, Np] for the last window (ddpg.py:62-79)."""
        T, n, gamma = rewards.shape[0], self.n_step, self.discount_factor_gamma
        valid = T - n + 1
        assert valid >= 1, "the batch is shorter than n_step"
        done = done_flags.to(rewards.dtype)[:, :, None]
        # step `last = i + n - 1` of every window i
        last_r, last_d = rewards[n - 1:], done[n - 1:]
        r = torch.empty_like(last_r)
        if valid > 1:       # windows whose last step has a successor inside the batch
            r[:-1] = last_r[:-1] + (1 - last_d[:-1]) * gamma * boot
        r[-1] = last_d[-1] * last_r[-1] + (1 - last_d[-1]) * boot_last
        for j in range(1, n):
            lo = n - 1 - j
            r = (1 - done[lo:lo + valid]) * gamma * r + rewards[lo:lo + valid]
        return r

    def sampled_returns(self, rewards, done, boot):
        """The n-step returns [B] of B sampled windows: rewards and done flags [n_step, B] of
        each window's steps and its bootstrap value `boot` [B].  Every window is a regular one:
        R = r_0 + (1 - d_0) gamma (r_1 + ... (1 - d_{n-1}) gamma boot), with no last-window
        rule, in window_returns' operation order."""
        r = boot
        for j in reversed(range(self.n_step)):
            r = (1 - done[j]) * self.discount_factor_gamma * r + rewards[j]
        return r

    def compute_loss_and_metrics(self, timestep=None, actions_batch=None, rewards_batch=None,
                                 done_flags_batch=None, value_functions_batch=None,
                                 next_value_functions_batch=None, j_functions_batch=None,
                                 perform_logging=False):
        assert timestep is not None and actions_batch is not None
        assert rewards_batch is not None and done_flags_batch is not None
        assert value_functions_batch is not None and next_value_functions_batch is not None
        assert j_functions_batch is not None
        valid = rewards_batch.shape[0] - self.n_step + 1
        returns = self.n_step_returns(rewards_batch, done_flags_batch,
                                      next_value_functions_batch.detach())
        norm_returns = self._normalize(returns) if self.normalize_return else returns
        values = value_functions_batch[:valid]
        critic_loss = nn.functional.mse_loss(values, norm_returns)
        j_values = j_functions_batch[:valid]
        norm_j = self._normalize(j_values) if self.normalize_return else j_values
        actor_loss = -norm_j.mean()
        metrics = {}
        if perform_logging:
            metrics = self.loss_metrics(actor_loss.item(), critic_loss.item(), rewards_batch,
                                        actions_batch, values.detach(), j_values.detach(),
                                        returns)
        return actor_loss, critic_loss, metrics

    def loss_metrics(self, actor_loss, critic_loss, rewards_batch, actions_batch, values,
                     j_values, returns):
        """The logged metrics of one update: the losses as floats, values / j_values / returns
        over the loss rows [valid, E, Np]; shared by the torch loss above and the fused update
        (fused_ddpg.py)."""
        norm_returns = self._normalize(returns) if self.normalize_return else returns
        advantages = norm_returns - values
        norm_adv = self._normalize(advantages) if self.normalize_advantage else advantages
        var_expl = max(-1.0, float(1 - norm_adv.var() / (norm_returns.var() + _EPSILON)))
        metrics = {
            "Total loss": actor_loss + critic_loss,
            "Actor loss": actor_loss, "Critic loss": critic_loss,
            "Mean rewards": rewards_batch.mean().item(),
            "Max. rewards": rewards_batch.max().item(),
            "Min. rewards": rewards_batch.min().item(),
            "Mean value function": values.mean().item(),
            "Mean J function": j_values.mean().item(),
            "Mean advantages": advantages.mean().item(),
            "Mean (norm.) advantages": norm_adv.mean().item(),
            "Mean (discounted) returns": returns.mean().item(),
            "Mean normalized returns": norm_returns.mean().item(),
            "Variance explained by the value function": var_expl,
        }
        a = actions_batch.float()
        for k in range(a.shape[-1]):
            metrics.update({
                f"Std. of action_{k} over agents": a[..., k].std(dim=2).mean().item(),
                f"Std. of action_{k} over envs": a[..., k].std(dim=1).mean().item(),
                f"Std. of action_{k} over time": a[..., k].std(dim=0).mean().item(),
                f"Max of action_{k}": a[..., k].max().item(),
                f"Min of action_{k}": a[..., k].min().item(),
            })
        return metrics
