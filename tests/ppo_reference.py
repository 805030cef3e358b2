"""Float64 reference of the multi-epoch PPO kernels (wdb_gae, wdb_ppo_loss_and_grads,
wdb_ppo_gaussian_loss_and_grads in csrc/wdb_update.cu), in plain numpy.

Every float output is a (value, bar) pair as in update_reference.py: the float64 value of the
kernel's float32 operation sequence on its float32 inputs, and a running-error bound on how far
a correct float32 evaluation may lie from it (u = 2**-24 per rounding, logf 1 ulp, expf 2 ulp,
double sums with their own (n + 1) 2**-53 term).  The math:

  GAE, d = done > 0:  A[T-1] = d ? r - V : 0
                      A[t] = (r + (d ? 0 : gamma V[t+1])) - V + (d ? 0 : gl A[t+1]),  gl = fl(gamma lam)
                      value_target = A + V
  minibatch loss:     l = Categorical log-prob summed over heads (q = p / sum p, log of q clamped
                      to [eps, 1 - eps]) or the diagonal Normal log-prob;  rho = exp(l - l_old)
                      policy = -(1/B) sum min(rho A, clamp(rho, 1 - clip, 1 + clip) A)   (PPO)
                             = -(1/B) sum l A                                            (A2C)
                      loss = policy + vf (1/B) sum (V - vt)^2 - c (1/B) sum H
  gradients:          w = -B d policy / d l: A2C A; PPO g rho with g = A (x < y), A [rho in the
                      closed clip interval] (x > y), half of each on a tie x == y.

Where the kernel's branch depends on a computed value -- the clamp test of q, rho against the
clip interval, x against y -- the row is `decided` only if every float32 value within the bar
takes the same branch; the GPU tests compare gradients on decided rows (inputs are built so that
nearly all rows are) and the CPU tests check the torch semantics exactly at the boundaries.
With prob_eps = 2**-52 the same functions give the float64 math torch evaluates in float64.
"""
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from update_reference import (  # noqa: E402
    D, EPS32, TINY, UREL, _f32_ceil, _f32_floor, _rnd, exact, f_add, f_div, f_exp, f_log,
    f_mul, f_neg, f_sub, select, sum_double)

HALF_LOG_2PI = 0.91893853320467274178


def _f32(x):
    return np.float64(np.float32(x))


def _const(c):
    """A float32 constant of the kernel: its exact value and its representation error."""
    return np.float64(c), abs(_f32(c) - np.float64(c))


def gae(rewards, values, done, gamma, lam):
    """rewards / values [T, E, Np] float32, done [T, E] (> 0 = done), gamma / lam as the float32
    values the ABI carries -> (advantages, value_targets) as (value, bar) pairs."""
    T = rewards.shape[0]
    r64, v64 = rewards.astype(np.float64), values.astype(np.float64)
    d = np.broadcast_to((done > 0)[:, :, None], rewards.shape)
    g = exact(_f32(gamma))
    gl = (_f32(gamma) * _f32(lam), _rnd(_f32(gamma) * _f32(lam), 0.0))
    zero = exact(np.zeros(rewards.shape[1:]))
    adv_v, adv_b = np.empty_like(r64), np.empty_like(r64)
    a_last = f_sub(exact(r64[T - 1]), exact(v64[T - 1]))
    adv_v[T - 1] = np.where(d[T - 1], a_last[0], 0.0)
    adv_b[T - 1] = np.where(d[T - 1], a_last[1], 0.0)
    for t in range(T - 2, -1, -1):
        boot = select(d[t], zero, f_mul(g, exact(v64[t + 1])))
        delta = f_sub(f_add(exact(r64[t]), boot), exact(v64[t]))
        carry = select(d[t], zero, f_mul(gl, (adv_v[t + 1], adv_b[t + 1])))
        adv_v[t], adv_b[t] = f_add(delta, carry)
    adv = (adv_v, adv_b)
    return adv, f_add(adv, exact(v64))


def _weight(logp, old, adv, ppo, clip, cast=_f32):
    """rho, w and the row's policy term with bars, and whether the branch is decided."""
    rho = f_exp(f_sub(logp, exact(old)))
    A = exact(adv)
    if not ppo:
        return rho, A, f_neg(f_mul(logp, A)), np.ones(adv.shape, bool)
    lo, hi = cast(1.0 - cast(clip)), cast(1.0 + cast(clip))
    r, b = rho
    inside = (r >= lo) & (r <= hi)
    in_dec = (r - b >= lo) & (r + b <= hi)
    out_dec = (r + b < lo) | (r - b > hi)
    x = f_mul(rho, A)
    y = f_mul(exact(np.clip(r, lo, hi)), A)
    y = (y[0], np.where(inside, x[1], y[1]))           # clamp(rho) == rho inside
    x_lt_y = x[0] < y[0]
    sep = np.abs(x[0] - y[0]) > x[1] + y[1]
    zero_adv = adv == 0
    decided = zero_adv | in_dec | (out_dec & sep)
    # inside: x == y exactly in float32 (a tie): g = A / 2 + A / 2 = A
    g = np.where(zero_adv, 0.0, np.where(inside, adv, np.where(x_lt_y, adv, 0.0)))
    w = f_mul(exact(g), rho)
    term = (np.minimum(x[0], y[0]), np.maximum(x[1], y[1]))
    return rho, w, f_neg(term), decided


def _clip_count(rho, clip, cast=_f32):
    r, b = rho
    c = cast(clip)
    over = np.abs(r - 1.0) > c
    unsure = np.abs(np.abs(r - 1.0) - c) <= b + UREL * (1.0 + abs(r)) + TINY
    return int(over.sum()), int(unsure.sum())


def _row_sums(pol, dv, ent, old, logp, rho, clip, cast=_f32):
    sq = (dv[0] ** 2, 2.0 * np.abs(dv[0]) * dv[1] + dv[1] ** 2)
    kl = f_sub(exact(old), logp)
    return [sum_double(pol), sum_double(sq), sum_double(ent), sum_double(kl),
            _clip_count(rho, clip, cast)]


def ppo_loss(probs, values, actions, advantages, value_targets, old_log_prob, ppo, clip,
             vf_coeff, entropy_coeff, prob_eps=EPS32):
    """The outputs of wdb_ppo_loss_and_grads on one minibatch (every array already in minibatch
    order): probs list of [B, A_k] float32, values / advantages / value_targets / old_log_prob
    [B] float32, actions [B, n_heads] int.  Returns dict: logp, rho, grad_probs (list),
    grad_values, sums (policy, value, entropy, KL as (value, bar); clip as (count, unsure)),
    decided [B] bool."""
    B = values.shape[0]
    cast = _f32 if prob_eps == EPS32 else np.float64
    vf = cast(vf_coeff)
    c = exact(cast(entropy_coeff))
    inv_b = (1.0 / B, _rnd(1.0 / B, D / B))
    lo_eps, hi_eps = prob_eps, 1.0 - prob_eps
    decided = np.ones(B, bool)
    logp = exact(np.zeros(B))
    ent = exact(np.zeros(B))
    heads = []
    for k, pk in enumerate(probs):
        P = pk.astype(np.float64)
        A = P.shape[-1]
        z = exact(np.zeros(B))
        for j in range(A):
            z = f_add(z, exact(P[:, j]))
        inv_z = f_div(exact(np.ones(B)), z)
        cols = []
        for j in range(A):
            q = f_mul(exact(P[:, j]), inv_z)
            inside = (q[0] >= lo_eps) & (q[0] <= hi_eps)
            if prob_eps == EPS32:
                lo_q, hi_q = _f32_ceil(q[0] - q[1]), _f32_floor(q[0] + q[1])
            else:
                lo_q, hi_q = q[0] - q[1], q[0] + q[1]
            same = (((lo_q >= lo_eps) & (lo_q <= hi_eps)) == inside) & (
                ((hi_q >= lo_eps) & (hi_q <= hi_eps)) == inside)
            decided &= same
            qc = (np.clip(q[0], lo_eps, hi_eps), np.where(inside, q[1], 0.0))
            lq = f_log(qc)
            ent = f_sub(ent, f_mul(lq, q))
            cols.append((q, inside, lq))
            logp = select(actions[:, k] == j, f_add(logp, lq), logp)
        heads.append((P, z, inv_z, cols))
    rho, w, pol, dec_w = _weight(logp, old_log_prob.astype(np.float64),
                                 advantages.astype(np.float64), ppo, clip, cast)
    decided &= dec_w
    dv = f_sub(exact(values.astype(np.float64)), exact(value_targets.astype(np.float64)))
    grad_values = f_mul(f_mul(exact(2.0 * vf), dv), inv_b)
    grad_probs = []
    for k, (P, z, inv_z, cols) in enumerate(heads):
        A = P.shape[-1]
        S = exact(np.zeros(B))
        gqs = []
        for j, (q, inside, lq) in enumerate(cols):
            gq = f_mul(c, f_add(lq, exact(inside.astype(np.float64))))
            taken = (actions[:, k] == j) & inside
            with np.errstate(divide="ignore", invalid="ignore"):
                q_safe = (np.where(inside, q[0], 1.0), np.where(inside, q[1], 0.0))
                gq = select(taken, f_sub(gq, f_div(w, q_safe)), gq)
            S = f_add(S, f_mul(gq, q))
            gqs.append(gq)
        gv = np.stack([g[0] for g in gqs], -1), np.stack([g[1] for g in gqs], -1)
        gp = f_mul(f_mul(f_sub(gv, (S[0][:, None], S[1][:, None])), inv_b),
                   (inv_z[0][:, None], inv_z[1][:, None]))
        grad_probs.append(gp)
    sums = _row_sums(pol, dv, ent, old_log_prob.astype(np.float64), logp, rho, clip, cast)
    return dict(logp=logp, rho=rho, grad_probs=grad_probs, grad_values=grad_values, sums=sums,
                decided=decided, B=B)


def ppo_gaussian_loss(mean, log_std, values, actions, advantages, value_targets, old_log_prob,
                      ppo, clip, vf_coeff, entropy_coeff, float64=False):
    """The outputs of wdb_ppo_gaussian_loss_and_grads on one minibatch: mean / actions [B, A]
    float32, log_std [A], the rest as ppo_loss (float64: coefficients taken as given, the math
    torch evaluates in float64).  Returns dict: logp, rho, grad_mean, grad_log_std, grad_values,
    sums, decided."""
    B, A = mean.shape
    cast = np.float64 if float64 else _f32
    vf = cast(vf_coeff)
    inv_b = (1.0 / B, _rnd(1.0 / B, D / B))
    ls = log_std.astype(np.float64)
    h = _const(HALF_LOG_2PI)
    c_ent = _const(0.5 + HALF_LOG_2PI)
    ent = exact(np.zeros(B))
    logp = exact(np.zeros(B))
    zs, inv_stds = [], []
    for k in range(A):
        ent = f_add(ent, f_add(exact(np.full(B, ls[k])), (np.full(B, c_ent[0]),
                                                           np.full(B, c_ent[1]))))
        inv_std = f_exp(exact(np.full(B, -ls[k])))
        z = f_mul(f_sub(exact(actions[:, k].astype(np.float64)),
                        exact(mean[:, k].astype(np.float64))), inv_std)
        term = f_sub(f_sub(f_mul(f_mul(exact(-0.5), z), z), exact(np.full(B, ls[k]))),
                     (np.full(B, h[0]), np.full(B, h[1])))
        logp = f_add(logp, term)
        zs.append(z)
        inv_stds.append(inv_std)
    rho, w, pol, decided = _weight(logp, old_log_prob.astype(np.float64),
                                   advantages.astype(np.float64), ppo, clip, cast)
    dv = f_sub(exact(values.astype(np.float64)), exact(value_targets.astype(np.float64)))
    grad_values = f_mul(f_mul(exact(2.0 * vf), dv), inv_b)
    gm = [f_mul(f_mul(f_mul(f_neg(w), z), s), inv_b) for z, s in zip(zs, inv_stds)]
    grad_mean = (np.stack([g[0] for g in gm], -1), np.stack([g[1] for g in gm], -1))
    g_ls = []
    for z in zs:
        t = f_mul(w, f_sub(f_mul(z, z), exact(np.ones(B))))
        acc, bar = sum_double(t)
        v = -acc / B - cast(entropy_coeff)
        bar = bar / B + 4 * D * (abs(acc) / B + abs(cast(entropy_coeff)))
        g_ls.append((v, bar + UREL * (abs(v) + bar) + TINY))
    grad_log_std = (np.array([g[0] for g in g_ls]), np.array([g[1] for g in g_ls]))
    sums = _row_sums(pol, dv, ent, old_log_prob.astype(np.float64), logp, rho, clip, cast)
    return dict(logp=logp, rho=rho, grad_mean=grad_mean, grad_log_std=grad_log_std,
                grad_values=grad_values, sums=sums, decided=decided, B=B)


def loss_value(sums, B, vf_coeff, entropy_coeff):
    """fused_ppo_loss's loss: (policy + vf * value - c * entropy) / B in double, then float32."""
    (s0, b0), (s1, b1), (s2, b2) = sums[:3]
    v = (s0 + vf_coeff * s1 - entropy_coeff * s2) / B
    mag = (abs(s0) + b0 + abs(vf_coeff) * (abs(s1) + b1) + abs(entropy_coeff) * (abs(s2) + b2)) / B
    bar = (b0 + abs(vf_coeff) * b1 + abs(entropy_coeff) * b2) / B + 8 * D * mag
    return v, bar + UREL * (abs(v) + bar) + TINY


def fsum(x):
    return math.fsum(np.ravel(x).tolist())
