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


class _FusedGaussianPGLoss(torch.autograd.Function):
    """`wdb_pg_gaussian_loss_and_grads`: the same loss for a diagonal Gaussian policy (mean per
    row, state-independent log_std)."""

    @staticmethod
    def forward(ctx, values, actions, rewards, done, gamma, vf_coeff, entropy_coeff, ppo,
                want_returns, mean, log_std):
        T, E, Np = rewards.shape
        A = int(mean.shape[-1])
        assert mean.shape == (T, E, Np, A) and actions.shape == mean.shape
        assert log_std.shape == (A,)
        dev = rewards.device
        values_c = values.detach().contiguous().float()
        mean_c = mean.detach().contiguous().float()
        log_std_c = log_std.detach().contiguous().float()
        actions_c = actions.detach().contiguous().float()
        rewards_c = rewards.contiguous().float()
        done_c = (done > 0).to(torch.int32).contiguous()
        g_mean = torch.empty_like(mean_c)
        g_log_std = torch.empty_like(log_std_c)
        g_values = torch.empty_like(values_c)
        returns = torch.empty_like(rewards_c) if want_returns else None
        sums = torch.zeros(4, dtype=torch.float64, device=dev)
        n_ctas = -(-(E * Np) // _lib.PG_GAUSSIAN_ROWS_PER_CTA)
        partials = torch.empty((n_ctas, A), dtype=torch.float64, device=dev)
        L = _lib.PgGaussianLoss()
        L.T, L.n_envs, L.n_agents, L.action_dim = T, E, Np, A
        L.mean, L.log_std, L.values = _lib.ptr(mean_c), _lib.ptr(log_std_c), _lib.ptr(values_c)
        L.actions, L.rewards, L.done = _lib.ptr(actions_c), _lib.ptr(rewards_c), _lib.ptr(done_c)
        L.gamma, L.vf_coeff, L.entropy_coeff = float(gamma), float(vf_coeff), float(entropy_coeff)
        L.grad_mean, L.grad_log_std = _lib.ptr(g_mean), _lib.ptr(g_log_std)
        L.grad_values, L.returns = _lib.ptr(g_values), _lib.ptr(returns)
        L.sums, L.partials = _lib.ptr(sums), _lib.ptr(partials)
        _lib.check(_lib.load().wdb_pg_gaussian_loss_and_grads(_lib.stream_ptr(), ctypes.byref(L)),
                   "pg_gaussian_loss_and_grads")
        m = float(T) * E * Np
        policy = (-sums[3] if ppo else sums[0]) / m
        vf = sums[1] / m
        ent = sums[2] / m
        loss = (policy + vf_coeff * vf - entropy_coeff * ent).to(torch.float32)
        ctx.save_for_backward(g_values, g_mean, g_log_std)
        ctx.values_shape = values.shape
        parts = torch.stack([policy, vf, ent]).to(torch.float32)
        if returns is None:
            returns = torch.empty(0, device=dev)
        ctx.mark_non_differentiable(parts, returns)
        return loss, parts, returns

    @staticmethod
    def backward(ctx, grad_loss, _gp, _gr):
        g_values, g_mean, g_log_std = ctx.saved_tensors
        gv = (g_values * grad_loss).view(ctx.values_shape)
        return (gv, None, None, None, None, None, None, None, None, g_mean * grad_loss,
                g_log_std * grad_loss)


def fused_gaussian_pg_loss_supported(mean):
    """True if `wdb_pg_gaussian_loss_and_grads` takes this action dimension."""
    return bool(_lib.load().wdb_pg_gaussian_loss_supported(int(mean.shape[-1])))


def fused_gaussian_pg_loss(values, mean, log_std, actions, rewards, done, gamma, vf_coeff,
                           entropy_coeff, ppo=False, want_returns=False):
    """values [T,E,Np], mean [T,E,Np,A] and log_std [A] (require grad), float actions
    [T,E,Np,A], rewards [T,E,Np], done [T,E].  Returns as fused_pg_loss."""
    return _FusedGaussianPGLoss.apply(values, actions, rewards, done, gamma, vf_coeff,
                                      entropy_coeff, bool(ppo), bool(want_returns), mean, log_std)


# ---- multi-epoch PPO over minibatches: `wdb_ppo_loss_and_grads` /
# `wdb_ppo_gaussian_loss_and_grads` (csrc/wdb_update.cu) on one minibatch of B rows.  The model
# outputs arrive in minibatch order; actions, advantages, value targets and old log-probs stay
# in the flat [R] batch and the kernel reads them through the int32 row list.
def _ppo_loss_from_sums(sums, B, vf_coeff, entropy_coeff):
    return ((sums[0] + vf_coeff * sums[1] - entropy_coeff * sums[2]) / B).to(torch.float32)


class _FusedPPOLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, values, rows, batch, ppo, clip_param, vf_coeff, entropy_coeff, *probs):
        B = int(values.shape[0])
        dev = values.device
        L = _lib.PpoLoss()
        L.B, L.n_heads = B, len(probs)
        values_c = values.detach().contiguous().float()
        probs_c = [p.detach().contiguous().float() for p in probs]
        g_probs = [torch.empty_like(p) for p in probs_c]
        g_values = torch.empty_like(values_c)
        sums = torch.zeros(5, dtype=torch.float64, device=dev)
        for k, p in enumerate(probs_c):
            assert p.shape[0] == B
            L.n_actions[k] = int(p.shape[-1])
            L.probs[k] = _lib.ptr(p)
            L.grad_probs[k] = _lib.ptr(g_probs[k])
        L.values, L.rows, L.actions = _lib.ptr(values_c), _lib.ptr(rows), _lib.ptr(batch.actions)
        L.advantages, L.value_targets = _lib.ptr(batch.advantages), _lib.ptr(batch.value_targets)
        L.old_log_prob = _lib.ptr(batch.old_log_prob)
        L.ppo, L.clip_param = int(ppo), float(clip_param)
        L.vf_coeff, L.entropy_coeff = float(vf_coeff), float(entropy_coeff)
        L.grad_values, L.sums = _lib.ptr(g_values), _lib.ptr(sums)
        _lib.check(_lib.load().wdb_ppo_loss_and_grads(_lib.stream_ptr(), ctypes.byref(L)),
                   "ppo_loss_and_grads")
        ctx.save_for_backward(g_values, *g_probs)
        ctx.mark_non_differentiable(sums)
        return _ppo_loss_from_sums(sums, B, vf_coeff, entropy_coeff), sums

    @staticmethod
    def backward(ctx, grad_loss, _gs):
        g_values, *g_probs = ctx.saved_tensors
        return (g_values * grad_loss, None, None, None, None, None, None,
                *[g * grad_loss for g in g_probs])


class _FusedPPOGaussianLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, values, rows, batch, ppo, clip_param, vf_coeff, entropy_coeff, mean,
                log_std):
        B, A = int(mean.shape[0]), int(mean.shape[-1])
        assert mean.shape == (B, A) and log_std.shape == (A,) and values.shape == (B,)
        dev = values.device
        values_c = values.detach().contiguous().float()
        mean_c = mean.detach().contiguous().float()
        log_std_c = log_std.detach().contiguous().float()
        g_mean = torch.empty_like(mean_c)
        g_log_std = torch.empty_like(log_std_c)
        g_values = torch.empty_like(values_c)
        sums = torch.zeros(5, dtype=torch.float64, device=dev)
        partials = torch.empty((-(-B // _lib.PG_GAUSSIAN_ROWS_PER_CTA), A), dtype=torch.float64,
                               device=dev)
        L = _lib.PpoGaussianLoss()
        L.B, L.action_dim = B, A
        L.mean, L.log_std, L.values = _lib.ptr(mean_c), _lib.ptr(log_std_c), _lib.ptr(values_c)
        L.rows, L.actions = _lib.ptr(rows), _lib.ptr(batch.actions)
        L.advantages, L.value_targets = _lib.ptr(batch.advantages), _lib.ptr(batch.value_targets)
        L.old_log_prob = _lib.ptr(batch.old_log_prob)
        L.ppo, L.clip_param = int(ppo), float(clip_param)
        L.vf_coeff, L.entropy_coeff = float(vf_coeff), float(entropy_coeff)
        L.grad_mean, L.grad_log_std = _lib.ptr(g_mean), _lib.ptr(g_log_std)
        L.grad_values, L.sums, L.partials = _lib.ptr(g_values), _lib.ptr(sums), _lib.ptr(partials)
        _lib.check(_lib.load().wdb_ppo_gaussian_loss_and_grads(_lib.stream_ptr(),
                                                               ctypes.byref(L)),
                   "ppo_gaussian_loss_and_grads")
        ctx.save_for_backward(g_values, g_mean, g_log_std)
        ctx.mark_non_differentiable(sums)
        return _ppo_loss_from_sums(sums, B, vf_coeff, entropy_coeff), sums

    @staticmethod
    def backward(ctx, grad_loss, _gs):
        g_values, g_mean, g_log_std = ctx.saved_tensors
        return (g_values * grad_loss, None, None, None, None, None, None, g_mean * grad_loss,
                g_log_std * grad_loss)


def fused_ppo_loss_supported(probs, log_std=None):
    """True if the minibatch kernel takes these heads (Categorical) or this action dimension
    (Gaussian: log_std given, probs = [mean])."""
    L = _lib.load()
    if log_std is not None:
        return bool(L.wdb_ppo_gaussian_loss_supported(int(probs[0].shape[-1])))
    widths = [int(p.shape[-1]) for p in probs]
    arr = (ctypes.c_int * max(1, len(widths)))(*widths)
    return bool(L.wdb_ppo_loss_supported(len(widths), arr))


def fused_ppo_loss(values, probs, rows, batch, ppo, clip_param, vf_coeff, entropy_coeff,
                   log_std=None):
    """values [B] and probs (list of [B, A_k], or [mean [B, A]] with log_std [A]) require grad;
    rows int32 [B] into the flat batch; batch has the flat `actions` (int32 [R, n_heads] or
    float [R, A]), `advantages`, `value_targets` and `old_log_prob` [R].  Returns (loss,
    float64 sums [5]: policy, value, entropy, KL, clip count)."""
    if log_std is not None:
        return _FusedPPOGaussianLoss.apply(values, rows, batch, bool(ppo), clip_param, vf_coeff,
                                           entropy_coeff, probs[0], log_std)
    return _FusedPPOLoss.apply(values, rows, batch, bool(ppo), clip_param, vf_coeff,
                               entropy_coeff, *probs)


def fused_log_prob(probs, actions, log_std=None):
    """The log-prob pre-pass: the same kernel, no old log-prob and no gradients, over the
    whole flat batch in order.  probs [R, A_k] per head (or [mean [R, A]] with log_std),
    actions as fused_ppo_loss.  Returns float32 [R]."""
    R = int(probs[0].shape[0])
    out = torch.empty(R, dtype=torch.float32, device=probs[0].device)
    probs_c = [p.detach().contiguous().float() for p in probs]
    if log_std is not None:
        L = _lib.PpoGaussianLoss()
        L.B, L.action_dim = R, int(probs_c[0].shape[-1])
        L.mean, L.log_std = _lib.ptr(probs_c[0]), _lib.ptr(log_std.detach().contiguous().float())
        L.actions, L.log_prob = _lib.ptr(actions), _lib.ptr(out)
        _lib.check(_lib.load().wdb_ppo_gaussian_loss_and_grads(_lib.stream_ptr(),
                                                               ctypes.byref(L)), "ppo_log_prob")
        return out
    L = _lib.PpoLoss()
    L.B, L.n_heads = R, len(probs_c)
    for k, p in enumerate(probs_c):
        L.n_actions[k] = int(p.shape[-1])
        L.probs[k] = _lib.ptr(p)
    L.actions, L.log_prob = _lib.ptr(actions), _lib.ptr(out)
    _lib.check(_lib.load().wdb_ppo_loss_and_grads(_lib.stream_ptr(), ctypes.byref(L)),
               "ppo_log_prob")
    return out
