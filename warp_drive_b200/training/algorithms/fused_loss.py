"""Fused A2C / PPO loss: `wdb_pg_loss_and_grads` (csrc/wdb_update.cu) wrapped as an autograd
function.  One kernel computes returns, advantages, log-probs, entropies, the loss sums and
the gradient of the total loss with respect to the model outputs; autograd only has to run
the MLP's backward from there (reference: a2c.py:80-130 / ppo.py:82-141 as ~100 torch ops)."""
import ctypes

import torch

from warp_drive_b200 import lib as _lib


class _FusedPGLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, values, actions, rewards, done, gamma, vf_coeff, entropy_coeff, ppo,
                want_returns, *probs):
        T, E, Np = rewards.shape
        L = _lib.PgLoss()
        L.T, L.n_envs, L.n_agents, L.n_heads = T, E, Np, len(probs)
        values_c = values.detach().contiguous().float()
        probs_c = [p.detach().contiguous().float() for p in probs]
        actions_c = actions.contiguous().to(torch.int32)
        rewards_c = rewards.contiguous().float()
        done_c = (done > 0).to(torch.int32).contiguous()
        g_probs = [torch.empty_like(p) for p in probs_c]
        g_values = torch.empty_like(values_c)
        returns = torch.empty_like(rewards_c) if want_returns else None
        sums = torch.zeros(4, dtype=torch.float64, device=rewards.device)
        for k, p in enumerate(probs_c):
            assert p.shape[:3] == (T, E, Np)
            L.n_actions[k] = int(p.shape[-1])
            L.probs[k] = _lib.ptr(p)
            L.grad_probs[k] = _lib.ptr(g_probs[k])
        L.values, L.actions = _lib.ptr(values_c), _lib.ptr(actions_c)
        L.rewards, L.done = _lib.ptr(rewards_c), _lib.ptr(done_c)
        L.gamma, L.vf_coeff, L.entropy_coeff = float(gamma), float(vf_coeff), float(entropy_coeff)
        L.grad_values = _lib.ptr(g_values)
        L.returns = _lib.ptr(returns)
        L.sums = _lib.ptr(sums)
        _lib.check(_lib.load().wdb_pg_loss_and_grads(_lib.stream_ptr(), ctypes.byref(L)),
                   "pg_loss_and_grads")
        m = float(T) * E * Np
        policy = (-sums[3] if ppo else sums[0]) / m
        vf = sums[1] / m
        ent = sums[2] / m
        loss = (policy + vf_coeff * vf - entropy_coeff * ent).to(torch.float32)
        ctx.save_for_backward(g_values, *g_probs)
        ctx.values_shape = values.shape
        parts = torch.stack([policy, vf, ent]).to(torch.float32)
        if returns is None:
            returns = torch.empty(0, device=rewards.device)
        ctx.mark_non_differentiable(parts, returns)
        return loss, parts, returns

    @staticmethod
    def backward(ctx, grad_loss, _gp, _gr):
        g_values, *g_probs = ctx.saved_tensors
        gv = (g_values * grad_loss).view(ctx.values_shape)
        return (gv, None, None, None, None, None, None, None, None,
                *[g * grad_loss for g in g_probs])


def fused_pg_loss_supported(probs):
    """True if `wdb_pg_loss_and_grads` takes these heads (the library's own launch check)."""
    widths = [int(p.shape[-1]) for p in probs]
    arr = (ctypes.c_int * max(1, len(widths)))(*widths)
    return bool(_lib.load().wdb_pg_loss_supported(len(widths), arr))


def fused_pg_loss(values, probs, actions, rewards, done, gamma, vf_coeff, entropy_coeff,
                  ppo=False, want_returns=False):
    """values [T,E,Np] (requires grad), probs: list of [T,E,Np,A_k] (require grad), actions
    [T,E,Np,n_heads], rewards [T,E,Np], done [T,E].  Returns (loss, (policy_loss, vf_loss,
    mean_entropy) tensor, returns or empty tensor)."""
    return _FusedPGLoss.apply(values, actions, rewards, done, gamma, vf_coeff, entropy_coeff,
                              bool(ppo), bool(want_returns), *probs)
