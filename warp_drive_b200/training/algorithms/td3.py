"""TD3 objective (Fujimoto, van Hoof and Meger, "Addressing Function Approximation Error in
Actor-Critic Methods", ICML 2018) on DDPG's replay ring and n-step returns: twin critics with
the minimum of the two target critics in the bootstrap, clipped Gaussian noise on the target
policy's action, and the actor (with the targets) updated every `policy_delay` critic updates.

Per window i of the ring (the loss rows of DDPG, `valid = T - n_step + 1` windows):
    a' = clamp(pi'(s') + clamp(sigma scale eps, -c scale, c scale), bias - scale, bias + scale)
    R  = DDPG's n-step return bootstrapped with min(Q1'(s', a'), Q2'(s', a')) at DDPG's
         bootstrap slot (the last window: the ring's last slot, undiscounted)
    critic loss = mse(Q1(s, a), R) + mse(Q2(s, a), R)      (reaches only the two critics)
    actor loss  = -mean Q1(s, pi(s))                         (reaches only the actor)
eps ~ N(0, 1) is one draw per (loss row, action dim) per update; sigma (`target_noise`) and c
(`target_noise_clip`) are in units of the actor's action scale, as in the paper.
"""
import torch
from torch import nn

from warp_drive_b200.training.algorithms.ddpg import DDPG, _EPSILON


class TD3(DDPG):
    # TrainerTD3 runs this policy's update as native kernels (fused_td3.py) when the shapes
    # allow it; False keeps the torch autograd update (a test switch, not a config key)
    use_fused_update = True

    def __init__(self, discount_factor_gamma=1.0, normalize_advantage=False,
                 normalize_return=False, n_step=1, target_noise=0.2, target_noise_clip=0.5,
                 policy_delay=2):
        if normalize_return:
            raise ValueError("TD3 does not normalise returns (normalize_return: True)")
        if int(policy_delay) != policy_delay or policy_delay < 1:
            raise ValueError(f"policy_delay must be an integer >= 1, got {policy_delay}")
        if target_noise < 0 or target_noise_clip < 0:
            raise ValueError("target_noise and target_noise_clip must be >= 0, got "
                             f"{target_noise} and {target_noise_clip}")
        super().__init__(discount_factor_gamma, normalize_advantage, False, n_step)
        self.target_noise = float(target_noise)
        self.target_noise_clip = float(target_noise_clip)
        self.policy_delay = int(policy_delay)

    def bootstrap_slots(self, T):
        """The ring slot (time order) whose observation bootstraps each window."""
        valid = T - self.n_step + 1
        return [i + self.n_step if i < valid - 1 else T - 1 for i in range(valid)]

    def target_actions(self, target_pi, noise, scale, bias):
        """a' from the target actor's actions [..., A] and standard normal noise of the same
        shape."""
        lim = self.target_noise_clip * scale
        eps = (noise * (self.target_noise * scale)).clamp(-lim, lim)
        return (target_pi + eps).clamp(bias - scale, bias + scale)

    def returns(self, rewards, done_flags, boot):
        """n-step returns [valid, E, Np] from the per-window bootstrap values `boot` [valid,
        E, Np] (already the minimum of the two target critics)."""
        return self.window_returns(rewards, done_flags, boot[:-1], boot[-1])

    @staticmethod
    def critic_losses(q1, q2, returns):
        return nn.functional.mse_loss(q1, returns), nn.functional.mse_loss(q2, returns)

    @staticmethod
    def actor_loss(j_values):
        return -j_values.mean()

    @staticmethod
    def actor_metrics(actor_loss):
        """The actor's logged metrics, on an update that stepped it."""
        return {"Actor loss": actor_loss, "Mean J function": -actor_loss}

    def loss_metrics(self, critic1_loss, critic2_loss, rewards_batch, actions_batch, q1_values,
                     returns):
        """The logged critic metrics of one update: the losses as floats, Q1 and the returns
        over the loss rows [valid, E, Np].  Shared by the torch and the fused update
        (fused_td3.py)."""
        advantages = returns - q1_values
        norm_adv = self._normalize(advantages) if self.normalize_advantage else advantages
        var_expl = max(-1.0, float(1 - norm_adv.var() / (returns.var() + _EPSILON)))
        metrics = {
            "Critic loss": critic1_loss + critic2_loss,
            "Critic 1 loss": critic1_loss, "Critic 2 loss": critic2_loss,
            "Mean rewards": rewards_batch.mean().item(),
            "Max. rewards": rewards_batch.max().item(),
            "Min. rewards": rewards_batch.min().item(),
            "Mean value function": q1_values.mean().item(),
            "Mean advantages": advantages.mean().item(),
            "Mean (discounted) returns": returns.mean().item(),
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


def torch_critic_loss(algo, target_actor, target_critic, target_critic2, critic, critic2, obs,
                      actions, rewards, done_flags, noise, boot_index):
    """Both critic losses by torch over the time-ordered ring: obs [T, E, Np, F], actions
    [T, E, Np, A], rewards [T, E, Np], done_flags [T, E], noise [valid, E, Np, A], boot_index
    the bootstrap slots (TD3.bootstrap_slots) as a device index tensor.  Returns (loss 1,
    loss 2, Q1, Q2, returns); only the two critics take gradients."""
    valid = noise.shape[0]
    with torch.no_grad():
        ob = obs.index_select(0, boot_index)
        pi = torch.cat(list(target_actor(obs=ob)), dim=-1)
        a_t = algo.target_actions(pi, noise, float(target_actor.action_scale),
                                  float(target_actor.action_bias))
        boot = torch.minimum(target_critic(obs=ob, action=a_t),
                             target_critic2(obs=ob, action=a_t))
        returns = algo.returns(rewards, done_flags, boot)
    q1 = critic(obs=obs[:valid], action=actions[:valid])
    q2 = critic2(obs=obs[:valid], action=actions[:valid])
    l1, l2 = algo.critic_losses(q1, q2, returns)
    return l1, l2, q1, q2, returns


def torch_sampled_critic_loss(algo, target_actor, target_critic, target_critic2, critic, critic2,
                              obs, actions, rewards, done, boot_obs, noise):
    """torch_critic_loss over B sampled windows gathered from the replay buffer: obs and
    boot_obs [B, F], actions [B, A], rewards and done [n_step, B], noise [B, A]."""
    with torch.no_grad():
        pi = torch.cat(list(target_actor(obs=boot_obs)), dim=-1)
        a_t = algo.target_actions(pi, noise, float(target_actor.action_scale),
                                  float(target_actor.action_bias))
        boot = torch.minimum(target_critic(obs=boot_obs, action=a_t),
                             target_critic2(obs=boot_obs, action=a_t))
        returns = algo.sampled_returns(rewards, done, boot)
    q1, q2 = critic(obs=obs, action=actions), critic2(obs=obs, action=actions)
    l1, l2 = algo.critic_losses(q1, q2, returns)
    return l1, l2, q1, q2, returns


def torch_actor_loss(algo, actor, critic, obs_rows):
    """-mean Q1(s, pi(s)) over the loss rows' observations [valid, E, Np, F]; returns (loss,
    J).  Call .backward(inputs=actor parameters) to keep the critic's gradient out."""
    j = critic(obs=obs_rows, action=actor(obs=obs_rows))
    return algo.actor_loss(j), j
