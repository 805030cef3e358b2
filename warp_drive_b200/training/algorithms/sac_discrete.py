"""Discrete-action SAC (Christodoulou, "Soft Actor-Critic for Discrete Action Settings", 2019) on
the replay buffer's sampled n-step windows: a categorical actor (`fully_connected_actor` on one
Discrete(A) head, its logits z), twin Q critics (`fully_connected_q`, A action values each) with
their targets, and SAC's temperature alpha = exp(log_alpha) tuned toward a target entropy.  There
is no target actor.

The torch statement of wdb_sac_discrete_{critic,actor}_update_sampled (include/wdb200.h), which
TrainerDiscreteSAC runs for the shapes the native passes do not take; tests/
sac_discrete_reference.py restates both passes in float64 NumPy.  Per sampled window g:
    log pi' = log_softmax(z(obs'))          (never log of a softmax: pi'_a = 0 adds 0)
    V'      = sum_a pi'_a (min(Q1', Q2')(obs')_a - alpha log pi'_a)
    R       = DQN's n-step return from V'   (every non-zero done flag ends the window)
    critic loss = mse(Q1(obs)[a], R) + mse(Q2(obs)[a], R)     (reaches only the two critics)
    actor loss  = (1/B) sum_g sum_a pi_a (alpha log pi_a - min(Q1, Q2)(obs)_a)
                                                               (reaches only the actor)
    d loss / d log_alpha = -((1/B) sum_g sum_a pi_a log pi_a + target_entropy)
The expectation over actions is exact, so there is no sampling noise in either pass.  The
default target entropy is 0.98 log A, the paper's.
"""
import math

import torch
from torch.nn import functional as func

from warp_drive_b200.training.algorithms.dqn import DQN
from warp_drive_b200.training.algorithms.sac import SAC


class DiscreteSAC(SAC):
    """SAC's temperature and alpha gradient with the exact expectation over A actions, DQN's
    terminal rule in the n-step return, and the discrete policy's metrics."""

    def __init__(self, discount_factor_gamma=1.0, normalize_advantage=False,
                 normalize_return=False, n_step=1, alpha=0.2, autotune_alpha=True,
                 target_entropy=None, n_actions=2):
        if int(n_actions) != n_actions or n_actions < 2:
            raise ValueError(f"discrete SAC needs at least 2 actions, got {n_actions}")
        if target_entropy is None:
            target_entropy = 0.98 * math.log(n_actions)
        super().__init__(discount_factor_gamma, normalize_advantage, normalize_return, n_step,
                         alpha=alpha, autotune_alpha=autotune_alpha,
                         target_entropy=target_entropy, action_dim=n_actions)

    def sampled_returns(self, rewards, done, boot):
        """DQN's n-step return: any non-zero done flag (MountainCar's 2 included) is terminal."""
        return DQN.sampled_returns(self, rewards, done, boot)

    @staticmethod
    def critic_metrics(critic1_loss, critic2_loss, mean_q1, returns):
        """The logged critic metrics of one update: the losses and the mean Q1(obs, a) as
        floats, the mean of the returns [B]."""
        return {"Critic loss": critic1_loss + critic2_loss, "Critic 1 loss": critic1_loss,
                "Critic 2 loss": critic2_loss, "Mean Q value": float(mean_q1),
                "Mean return": float(returns.double().mean())}


def actor_logits(actor, obs):
    """The logits [..., A] of a FullyConnectedActor's one softmax head."""
    x = obs
    for i in range(len(actor.fc)):
        x = actor.fc[str(i)](x)
    return actor.policy_head[0](x)


def torch_sampled_critic_loss(algo, actor, target_critic, target_critic2, critic, critic2,
                              log_alpha, obs, actions, rewards, done, boot_obs):
    """Both critic losses over B sampled windows: obs and boot_obs [B, F], int actions [B, 1],
    rewards and done [n_step, B].  Returns (loss 1, loss 2, Q1 [B], Q2 [B], returns [B]); only
    the two critics take gradients."""
    with torch.no_grad():
        log_pi = func.log_softmax(actor_logits(actor, boot_obs), dim=-1)
        q_t = torch.minimum(target_critic.q_values(boot_obs), target_critic2.q_values(boot_obs))
        boot = (log_pi.exp() * (q_t - log_alpha.exp() * log_pi)).sum(dim=-1)
        returns = algo.sampled_returns(rewards, done, boot)
    a = actions.long().reshape(-1, 1)
    q1 = critic.q_values(obs).gather(-1, a)[..., 0]
    q2 = critic2.q_values(obs).gather(-1, a)[..., 0]
    l1, l2 = algo.critic_losses(q1, q2, returns)
    return l1, l2, q1, q2, returns


def torch_actor_loss(algo, actor, critic, critic2, log_alpha, obs_rows):
    """(1/B) sum_g sum_a pi_a (alpha log pi_a - min(Q1, Q2)_a) over obs_rows [B, F]; returns
    (loss, sum_a pi_a min(Q1, Q2)_a [B], sum_a pi_a log pi_a [B]).  Call
    .backward(inputs=actor parameters) to keep the critics' and log_alpha's gradients out."""
    log_pi = func.log_softmax(actor_logits(actor, obs_rows), dim=-1)
    pi = log_pi.exp()
    with torch.no_grad():
        m = torch.minimum(critic.q_values(obs_rows), critic2.q_values(obs_rows))
    loss = (pi * (log_alpha.detach().exp() * log_pi - m)).sum(dim=-1).mean()
    return loss, (pi * m).sum(dim=-1).detach(), (pi * log_pi).sum(dim=-1).detach()
