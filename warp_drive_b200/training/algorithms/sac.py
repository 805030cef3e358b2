"""SAC objective (Haarnoja et al., "Soft Actor-Critic Algorithms and Applications", 2018) on
DDPG's replay ring and n-step returns: a tanh-squashed Gaussian actor (FullyConnectedSACActor),
twin critics and their targets, an entropy bonus with temperature alpha = exp(log_alpha), and
log_alpha tuned toward a target entropy.  SAC has no target actor.

Per window i of the ring (the loss rows of DDPG, `valid = T - n_step + 1` windows), with fresh
standard normals eps' (critic) and eps (actor) per update:
    a' = squash(mu(s') + sigma(s') eps'),  s' = DDPG's bootstrap slot
    R  = DDPG's n-step return bootstrapped with min(Q1'(s', a'), Q2'(s', a')) - alpha log pi(a'|s')
    critic loss = mse(Q1(s, a), R) + mse(Q2(s, a), R)            (reaches only the two critics)
    a  = squash(mu(s) + sigma(s) eps)
    actor loss  = mean(alpha log pi(a|s) - min(Q1, Q2)(s, a))     (reaches only the actor; ties
                                                                  of the minimum go to Q1)
    d loss / d log_alpha = -mean(log pi(a|s) + target_entropy)    (log pi detached)
log pi is the squashed density over tanh(u) in (-1, 1) (models/fully_connected_actor_critic.py,
`squashed_log_prob`): the action scale does not enter it, so the default target entropy is -A
whatever the action range.
"""
import math

import torch

from warp_drive_b200.training.algorithms.td3 import TD3


class SAC(TD3):
    """TD3's ring bookkeeping (bootstrap slots, window returns, critic losses and metrics) with
    SAC's bootstrap value and actor loss.  TD3's target-noise and delay settings do not apply."""

    def __init__(self, discount_factor_gamma=1.0, normalize_advantage=False,
                 normalize_return=False, n_step=1, alpha=0.2, autotune_alpha=True,
                 target_entropy=None, action_dim=1):
        if normalize_return:
            raise ValueError("SAC does not normalise returns (normalize_return: True)")
        if not alpha > 0:
            raise ValueError(f"alpha must be > 0, got {alpha}")
        if target_entropy is None:
            target_entropy = -float(action_dim)
        if not math.isfinite(float(target_entropy)):
            raise ValueError(f"target_entropy must be finite, got {target_entropy}")
        super().__init__(discount_factor_gamma, normalize_advantage, False, n_step,
                         target_noise=0.0, target_noise_clip=0.0, policy_delay=1)
        self.alpha = float(alpha)
        self.autotune_alpha = bool(autotune_alpha)
        self.target_entropy = float(target_entropy)

    def alpha_grad(self, sum_log_pi, rows):
        """d loss / d log_alpha from the actor pass's sum of log pi over `rows` loss rows (a
        device scalar: no host sync)."""
        return -(sum_log_pi / rows + self.target_entropy)

    @staticmethod
    def actor_metrics(actor_loss, mean_log_pi, alpha, alpha_loss):
        """The actor's and the temperature's logged metrics."""
        return {"Actor loss": actor_loss, "Entropy": -mean_log_pi, "Alpha": alpha,
                "Alpha loss": alpha_loss}


def min_first(q1, q2):
    """min(q1, q2) with ties to q1: the gradient goes to exactly one critic per row."""
    return torch.where(q1 <= q2, q1, q2)


def torch_critic_loss(algo, actor, target_critic, target_critic2, critic, critic2, log_alpha,
                      obs, actions, rewards, done_flags, noise, boot_index):
    """Both critic losses by torch over the time-ordered ring: obs [T, E, Np, F], actions
    [T, E, Np, A], rewards [T, E, Np], done_flags [T, E], noise [valid, E, Np, A] (eps'),
    boot_index the bootstrap slots (TD3.bootstrap_slots) as a device index tensor.  Returns
    (loss 1, loss 2, Q1, Q2, returns); only the two critics take gradients."""
    valid = noise.shape[0]
    with torch.no_grad():
        ob = obs.index_select(0, boot_index)
        a_t, log_pi = actor.sample(ob, noise)
        q_t = torch.minimum(target_critic(obs=ob, action=a_t), target_critic2(obs=ob, action=a_t))
        boot = q_t - log_alpha.exp() * log_pi
        returns = algo.returns(rewards, done_flags, boot)
    q1 = critic(obs=obs[:valid], action=actions[:valid])
    q2 = critic2(obs=obs[:valid], action=actions[:valid])
    l1, l2 = algo.critic_losses(q1, q2, returns)
    return l1, l2, q1, q2, returns


def torch_sampled_critic_loss(algo, actor, target_critic, target_critic2, critic, critic2,
                              log_alpha, obs, actions, rewards, done, boot_obs, noise):
    """torch_critic_loss over B sampled windows gathered from the replay buffer: obs and
    boot_obs [B, F], actions [B, A], rewards and done [n_step, B], noise [B, A] (eps')."""
    with torch.no_grad():
        a_t, log_pi = actor.sample(boot_obs, noise)
        q_t = torch.minimum(target_critic(obs=boot_obs, action=a_t),
                            target_critic2(obs=boot_obs, action=a_t))
        returns = algo.sampled_returns(rewards, done, q_t - log_alpha.exp() * log_pi)
    q1, q2 = critic(obs=obs, action=actions), critic2(obs=obs, action=actions)
    l1, l2 = algo.critic_losses(q1, q2, returns)
    return l1, l2, q1, q2, returns


def torch_actor_loss(algo, actor, critic, critic2, log_alpha, obs_rows, noise):
    """mean(alpha log pi - min(Q1, Q2)) over the loss rows' observations [valid, E, Np, F] with
    eps = noise [valid, E, Np, A]; returns (loss, min Q, log pi).  Call
    .backward(inputs=actor parameters) to keep the critics' and log_alpha's gradients out."""
    a, log_pi = actor.sample(obs_rows, noise)
    q = min_first(critic(obs=obs_rows, action=a), critic2(obs=obs_rows, action=a))
    loss = (log_alpha.detach().exp() * log_pi - q).mean()
    return loss, q, log_pi
