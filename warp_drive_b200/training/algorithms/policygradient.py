"""A2C and PPO objectives for the on-policy update that consumes the rollout batch.

Same mathematics as the reference (warp_drive/training/algorithms/policygradient/
a2c.py:40-194, ppo.py:42-204): bootstrapped discounted returns computed backwards in time
with done masking, optional per-timestep normalisation of returns / advantages over
(env, agent), categorical log-prob + entropy over every action head, MSE value loss.
The backward-time recursion runs as ONE kernel (wdb_discounted_returns) instead of
~6 elementwise launches per timestep.
"""
import torch
from torch import nn
from torch.distributions import Categorical

from warp_drive_b200.training.algorithms.fused_loss import fused_pg_loss, fused_pg_loss_supported
from warp_drive_b200.training.utils.param_scheduler import ParamScheduler

_EPSILON = 1e-10


def discounted_returns(rewards, done_flags, values, gamma):
    """returns[T-1] = done*r + (1-done)*V ; returns[t] = r[t] + (1-done[t])*gamma*returns[t+1]
    (a2c.py:80-93).  rewards/values [T, E, Np] float32, done_flags [T, E] int."""
    if rewards.is_cuda:
        from warp_drive_b200 import lib as _lib

        rewards = rewards.contiguous()
        values = values.contiguous().float()
        done = (done_flags > 0).to(torch.int32).contiguous()
        out = torch.empty_like(rewards)
        T, E, Np = rewards.shape
        _lib.check(_lib.load().wdb_discounted_returns(
            _lib.stream_ptr(), _lib.ptr(rewards), _lib.ptr(done), _lib.ptr(values),
            _lib.ptr(out), T, E, Np, float(gamma)), "discounted_returns")
        return out
    # host tensors (unit tests of the loss math)
    done = (done_flags > 0).to(rewards.dtype)[:, :, None]
    out = torch.zeros_like(rewards)
    out[-1] = done[-1] * rewards[-1] + (1 - done[-1]) * values[-1]
    for t in range(rewards.shape[0] - 2, -1, -1):
        out[t] = rewards[t] + (1 - done[t]) * gamma * out[t + 1]
    return out


class _PolicyGradient:
    def __init__(self, discount_factor_gamma=1.0, normalize_advantage=False,
                 normalize_return=False, vf_loss_coeff=0.01, entropy_coeff=0.01,
                 clip_param=None):
        assert 0 <= discount_factor_gamma <= 1
        self.discount_factor_gamma = discount_factor_gamma
        self.normalize_advantage = normalize_advantage
        self.normalize_return = normalize_return
        self.vf_loss_coeff_schedule = ParamScheduler(vf_loss_coeff)
        self.entropy_coeff_schedule = ParamScheduler(entropy_coeff)
        self.clip_param = clip_param
        # CUDA: returns / advantages / log-prob / entropy / loss AND the gradient with respect
        # to the model outputs in one kernel (fused_loss.py); the torch expression below stays
        # as the float32 reference the GPU tests compare against (and for the normalised /
        # env-subsampled variants)
        self.use_fused_loss = True

    @staticmethod
    def _normalize(x):
        return (x - x.mean(dim=(1, 2), keepdim=True)) / (x.std(dim=(1, 2), keepdim=True) + _EPSILON)

    def _policy_loss(self, log_prob, advantages):
        raise NotImplementedError

    def compute_loss_and_metrics(self, timestep=None, actions_batch=None, rewards_batch=None,
                                 done_flags_batch=None, action_probabilities_batch=None,
                                 value_functions_batch=None, perform_logging=False,
                                 negative_positive_ratio=-1):
        assert timestep is not None
        n_pos = n_neg = None
        if negative_positive_ratio > 0:
            # sparse-goal envs (MountainCar: done == 2 marks "goal reached",
            # mountain_car_step_numba.py:66-70): keep every env that reached the goal in this
            # batch and at most ratio x as many of the others (a2c.py:58-69, 196-220)
            keep, n_pos, n_neg = self._sample_positive_negative_env_ids(
                done_flags_batch, negative_positive_ratio)
            if keep is not None:
                actions_batch = actions_batch[:, keep]
                rewards_batch = rewards_batch[:, keep]
                done_flags_batch = done_flags_batch[:, keep]
                action_probabilities_batch = [p[:, keep] for p in action_probabilities_batch]
                value_functions_batch = value_functions_batch[:, keep]
        if (self.use_fused_loss and value_functions_batch.is_cuda and n_pos is None
                and not self.normalize_return and not self.normalize_advantage
                and fused_pg_loss_supported(action_probabilities_batch)):
            return self._fused_loss_and_metrics(
                timestep, actions_batch, rewards_batch, done_flags_batch,
                action_probabilities_batch, value_functions_batch, perform_logging)
        values_detached = value_functions_batch.detach()
        returns = discounted_returns(rewards_batch, done_flags_batch, values_detached,
                                     self.discount_factor_gamma)
        norm_returns = self._normalize(returns) if self.normalize_return else returns
        vf_loss = nn.functional.mse_loss(value_functions_batch, norm_returns)
        advantages = norm_returns - values_detached
        norm_adv = self._normalize(advantages) if self.normalize_advantage else advantages

        log_prob, mean_entropy = 0.0, 0.0
        for k in range(actions_batch.shape[-1]):
            dist = Categorical(action_probabilities_batch[k])
            mean_entropy = mean_entropy + dist.entropy().mean()
            log_prob = log_prob + dist.log_prob(actions_batch[..., k])
        policy_loss = self._policy_loss(log_prob, norm_adv)
        vf_c = self.vf_loss_coeff_schedule.get_param_value(timestep)
        ent_c = self.entropy_coeff_schedule.get_param_value(timestep)
        loss = policy_loss + vf_c * vf_loss - ent_c * mean_entropy
        metrics = {}
        if perform_logging:
            var_expl = 1 - norm_adv.detach().var() / (norm_returns.detach().var() + _EPSILON)
            metrics = {
                "VF loss coefficient": vf_c, "Entropy coefficient": ent_c,
                "Total loss": loss.item(), "Policy loss": policy_loss.item(),
                "Value function loss": vf_loss.item(),
                "Mean rewards": rewards_batch.mean().item(),
                "Max. rewards": rewards_batch.max().item(),
                "Min. rewards": rewards_batch.min().item(),
                "Mean value function": value_functions_batch.mean().item(),
                "Mean advantages": advantages.mean().item(),
                "Mean (norm.) advantages": norm_adv.mean().item(),
                "Mean (discounted) returns": returns.mean().item(),
                "Mean normalized returns": norm_returns.mean().item(),
                "Mean entropy": mean_entropy.item(),
                "Variance explained by the value function": max(-1.0, var_expl.item()),
            }
            a = actions_batch.float()
            for k in range(a.shape[-1]):
                metrics[f"Std. of action_{k} over agents"] = a[..., k].std(dim=2).mean().item()
                metrics[f"Std. of action_{k} over envs"] = a[..., k].std(dim=1).mean().item()
                metrics[f"Std. of action_{k} over time"] = a[..., k].std(dim=0).mean().item()
            if n_pos is not None:
                metrics["Num of Positive Sampled Envs"] = n_pos
                metrics["Num of Negative Sampled Envs"] = n_neg
        return loss, metrics

    def _fused_loss_and_metrics(self, timestep, actions_batch, rewards_batch, done_flags_batch,
                                action_probabilities_batch, value_functions_batch,
                                perform_logging):
        vf_c = self.vf_loss_coeff_schedule.get_param_value(timestep)
        ent_c = self.entropy_coeff_schedule.get_param_value(timestep)
        loss, parts, returns = fused_pg_loss(
            value_functions_batch, list(action_probabilities_batch), actions_batch,
            rewards_batch, done_flags_batch, self.discount_factor_gamma, vf_c, ent_c,
            ppo=self.clip_param is not None, want_returns=perform_logging)
        metrics = {}
        if perform_logging:
            values = value_functions_batch.detach()
            advantages = returns - values
            var_expl = 1 - advantages.var() / (returns.var() + _EPSILON)
            policy_loss, vf_loss, mean_entropy = (float(x) for x in parts)
            metrics = {
                "VF loss coefficient": vf_c, "Entropy coefficient": ent_c,
                "Total loss": loss.item(), "Policy loss": policy_loss,
                "Value function loss": vf_loss,
                "Mean rewards": rewards_batch.mean().item(),
                "Max. rewards": rewards_batch.max().item(),
                "Min. rewards": rewards_batch.min().item(),
                "Mean value function": values.mean().item(),
                "Mean advantages": advantages.mean().item(),
                "Mean (norm.) advantages": advantages.mean().item(),
                "Mean (discounted) returns": returns.mean().item(),
                "Mean normalized returns": returns.mean().item(),
                "Mean entropy": mean_entropy,
                "Variance explained by the value function": max(-1.0, var_expl.item()),
            }
            a = actions_batch.float()
            for k in range(a.shape[-1]):
                metrics[f"Std. of action_{k} over agents"] = a[..., k].std(dim=2).mean().item()
                metrics[f"Std. of action_{k} over envs"] = a[..., k].std(dim=1).mean().item()
                metrics[f"Std. of action_{k} over time"] = a[..., k].std(dim=0).mean().item()
        return loss, metrics

    @staticmethod
    def _sample_positive_negative_env_ids(done_flags_batch, negative_positive_ratio):
        """(env index tensor or None when nothing is dropped, #positive, #negative kept)."""
        positives = (done_flags_batch == 2).any(dim=0)
        pos_ids = positives.nonzero(as_tuple=True)[0]
        neg_ids = (~positives).nonzero(as_tuple=True)[0]
        n_pos, total = int(pos_ids.numel()), int(done_flags_batch.shape[1])
        n_neg = int(n_pos * negative_positive_ratio)
        if n_pos == 0 or n_pos + n_neg >= total:
            return None, n_pos, int(neg_ids.numel())
        pick = torch.randperm(int(neg_ids.numel()), device=neg_ids.device)[:n_neg]
        return torch.cat((pos_ids, neg_ids[pick])), n_pos, n_neg


class A2C(_PolicyGradient):
    """Advantage actor-critic (a2c.py:123-130)."""

    def _policy_loss(self, log_prob, advantages):
        return (-log_prob * advantages).mean()


class PPO(_PolicyGradient):
    """Clipped-surrogate PPO exactly as the reference states it (ppo.py:127-136): the
    'old' log-prob is the detached current one (single epoch over the fresh batch)."""

    def __init__(self, clip_param=0.1, **kw):
        super().__init__(clip_param=clip_param, **kw)
        assert 0 <= clip_param <= 1

    def _policy_loss(self, log_prob, advantages):
        ratio = torch.exp(log_prob - log_prob.detach())
        clipped = torch.clamp(ratio, 1.0 - self.clip_param, 1.0 + self.clip_param)
        return -torch.minimum(ratio * advantages, clipped * advantages).mean()
