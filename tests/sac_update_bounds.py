"""Float64 reference with error bars of the SAC-family replay update passes:
wdb_sac_{critic,actor}_update_sampled (csrc/wdb_ddpg_update.cu), wdb_sac_discrete_{critic,actor}_
update_sampled (csrc/wdb_sac_discrete.cu) and wdb_tqc_{critic,actor}_update_sampled
(csrc/wdb_tqc.cu).

Every output comes as a pair (value, bar), as in q_update_bounds: the float64 value of the
operation on the kernel's float32 inputs, and a bound on how far a correct float32 evaluation can
lie from it.  The values are those of replay_update_reference.sac_*_sampled,
sac_discrete_reference and tqc_reference, which stay the statement of the objective; the bars
follow the kernels' float32 operations one by one, by update_reference's and q_update_bounds'
rules (u = 2**-24; expf 2 ulp, logf 1 ulp; a sum of n terms in any order n u sum|terms|; the
gradient accumulations through tile_depth) and these:
  * tanhf within 2 ulp, log1pf within 1 ulp, an fmaf one rounding of the exact a b + c;
  * torch's softplus, x > 20 ? x : log1p(exp(x)), as the continuous log1p(exp(x)): the jump
    log1p(exp(-x)) of the x branch is charged in the bar, so no premise;
  * the float32 constants log 2 and log(2 pi) / 2 of squashed_dim are charged their distance
    from the exact constants (the values use the exact ones);
  * alpha = expf(log_alpha) of the float32 log_alpha: the value exp(log_alpha), 2 ulp;
  * fminf, a clamp and an order statistic are 1-Lipschitz: the min and the k-th smallest of a
    row take the largest bar among their candidates.

Branch premises (per row, `ok`), where a decision reads a computed value:
  * the backward ReLU masks of every network whose gradient or input gradient is formed
    (q_update_bounds.relu); forwards that only feed a value use max(z, 0), 1-Lipschitz;
  * the log-std clamp's gate in the actor passes: |raw - lo| > bar and |raw - hi| > bar (a
    clamped column's log-std gradient is then exactly 0, bar 0); the critic passes use only
    the clamped value, which is continuous;
  * SAC's actor routes its gradient through argmin(Q1, Q2), ties to Q1: |Q1 - Q2| > bar1 + bar2.
    The critic bootstrap uses only the value of the min: no premise.
TQC's truncation needs none: the k-th order statistic of a row's 2N atoms moves by at most the
largest bar among them, so each kept atom takes that row-wise maximum as its bar.  Its quantile
weight |tau - 1{u < 0}| multiplies clamp(u, -1, 1) and the Huber term, both 0 at u = 0, so each
product is continuous in u: where |u| <= bar either weight may be taken, and the product's bar
is |w c| + 1.01 (|c| + bar_c), c the clamp or Huber term.

How tight: as q_update_bounds' docstring says, a gradient element's bar adds up its rows'
absolute contributions, so it pins small elements, signs and exact zeros, while for the large
elements of the deep layers it is looser than the 2e-4 norm-wise tests, which stay."""
import math

import numpy as np

from q_update_bounds import (D, _softmax_parts, _sum_bar, backward, double_mean, double_sum,
                             f_back, f_dot, f_round, f_sum, forward, nstep, norm_of, tile_depth)
from update_reference import U, UREL, _rnd, exact, f_add, f_div, f_exp, f_log, f_mul, f_sub

LN2_F32 = float(np.float32(0.69314718055994531))
HALF_LOG_2PI_F32 = float(np.float32(0.91893853320467274))


# ---------------------------------------------------------------- primitives
def f_tanh(x, ulps=2):
    """tanhf within 2 ulp: the input's bar through the largest slope 1 - tanh^2 on [x - b,
    x + b], then the rounding."""
    v = np.tanh(x[0])
    slope = 1.0 - np.tanh(np.maximum(np.abs(x[0]) - x[1], 0.0)) ** 2
    p = slope * x[1]
    return v, p + 2.0 * U * ulps * (np.abs(v) + p) + ulps * 2.0 ** -149


def f_log1p(x, ulps=1):
    """log1pf within 1 ulp, of x > -1 by more than its bar."""
    assert np.all(x[0] - x[1] > -1.0)
    v = np.log1p(x[0])
    p = x[1] / (1.0 + x[0] - x[1])
    return v, p + 2.0 * U * ulps * (np.abs(v) + p) + ulps * 2.0 ** -149


def f_fma(a, b, c):
    """fmaf(a, b, c): one rounding of the exact a b + c of the computed inputs."""
    v = a[0] * b[0] + c[0]
    return v, _rnd(v, np.abs(a[0]) * b[1] + np.abs(b[0]) * a[1] + a[1] * b[1] + c[1])


def f_min(x, y):
    """fminf: 1-Lipschitz, the larger bar."""
    return np.minimum(x[0], y[0]), np.maximum(x[1], y[1])


def f_softplus(x):
    """x > 20 ? x : log1pf(expf(x)) (torch's threshold) as the continuous log1p(exp(x)): where
    the computed x may lie above 20 the branch's gap log1p(exp(-x)) to the curve is charged."""
    v = np.logaddexp(0.0, x[0])
    xc = np.minimum(x[0], 20.0)
    curve = f_log1p(f_exp((xc, x[1])))[1] + (x[0] - xc)
    curve = np.where(x[0] - x[1] <= 20.0, curve, 0.0)
    branch = np.where(x[0] + x[1] > 20.0, x[1] + np.log1p(np.exp(-(x[0] - x[1]))), 0.0)
    return v, np.maximum(curve, branch) + 4 * D * v


def f_alpha(log_alpha):
    """expf(*log_alpha) of the float32 log_alpha."""
    la = float(np.float32(log_alpha))
    return f_exp(exact(la))


def squashed_dim(mu, raw, eps, lo, hi):
    """squashed_dim (wdb_sac_terms.cuh) operation by operation on head columns mu, raw [B, A]
    (value, bar) and float32 normals eps [B, A]: dict of sigma, u, y, term (value, bar), ls,
    in_range [B, A] and ok [B] (no raw log-std within its bar of lo or hi, unless exact)."""
    lo, hi = float(np.float32(lo)), float(np.float32(hi))
    eps = np.asarray(eps, np.float64)
    rv, rb = raw
    in_range = (rv >= lo) & (rv <= hi)
    ok = (((np.abs(rv - lo) > rb) & (np.abs(rv - hi) > rb)) | (rb == 0)).all(axis=1)
    ls = (np.clip(rv, lo, hi), np.where((rv - rb >= hi) | (rv + rb <= lo), 0.0, rb))
    sigma = f_exp(ls)
    u = f_fma(sigma, exact(eps), mu)
    y = f_tanh(u)
    sp = f_softplus((-2.0 * u[0], 2.0 * u[1]))
    ln2 = (math.log(2.0), abs(LN2_F32 - math.log(2.0)))
    corr = f_sub(f_sub(ln2, u), sp)
    corr = (2.0 * corr[0], 2.0 * corr[1])
    c = (0.5 * math.log(2 * math.pi), abs(HALF_LOG_2PI_F32 - 0.5 * math.log(2 * math.pi)))
    t = f_mul(exact(-0.5 * eps), exact(eps))
    term = f_sub(f_sub(f_sub(t, ls), c), corr)
    return {"sigma": sigma, "u": u, "y": y, "term": term, "ls": ls, "in_range": in_range,
            "ok": ok}


def sac_nstep(boot, rewards, done, gamma):
    """sampled_return's ret = ((1 - d) gamma) ret + r on boot [B, ...], each product and sum
    rounded; (1 - d) gamma is exact for the done flags 0, 1 and 2."""
    ret = boot
    g = float(np.float32(gamma))
    extra = (slice(None),) + (None,) * (boot[0].ndim - 1)
    for j in reversed(range(rewards.shape[0])):
        om = ((1.0 - np.asarray(done[j], np.float64)) * g)[extra]
        r = np.asarray(rewards[j], dtype=np.float64)[extra]
        ret = f_add(f_mul(exact(np.broadcast_to(om, ret[0].shape)), ret),
                    exact(np.broadcast_to(r, ret[0].shape)))
    return ret


def _cat(*xs):
    return (np.concatenate([x[0] for x in xs], axis=1),
            np.concatenate([x[1] for x in xs], axis=1))


def _col(x, c):
    return x[0][:, c], x[1][:, c]


def _rows(rows):
    obs, actions, rewards, done, boot = rows
    f = lambda a: np.asarray(a, np.float64)  # noqa: E731
    return exact(f(obs)), np.asarray(actions), f(rewards), np.asarray(done), exact(f(boot))


def _squashed_head(La, x, eps, lo, hi, decide):
    """The actor's head and squashed_dim.  A head column whose weight row is all zero is its
    bias exactly (each fmaf adds an exact 0): bar 0, so a raw log-std pinned at lo or hi is a
    decided branch."""
    z, inputs, ok = forward(La, x, decide)
    pinned = (La[-1][0] == 0).all(axis=1)
    z = (z[0], np.where(pinned[None, :], 0.0, z[1]))
    A = z[0].shape[1] // 2
    s = squashed_dim((z[0][:, :A], z[1][:, :A]), (z[0][:, A:], z[1][:, A:]), eps, lo, hi)
    return s, inputs, ok


def _action(s, scale, bias):
    """__fadd_rn(__fmul_rn(scale, y), bias)."""
    return f_add(f_mul(exact(float(np.float32(scale))), s["y"]), exact(float(np.float32(bias))))


def _mse_grad(q, ret, B):
    e = f_sub(q, ret)
    d = f_mul(e, norm_of(B / 2.0))
    sq = (e[0] ** 2, 2 * np.abs(e[0]) * e[1] + e[1] ** 2 + D * e[0] ** 2)
    return e, d, double_sum(sq, 16)


def input_grad(L, inputs, d, first):
    """The gradient at the columns [first, in) of layer 0's input from the head delta d (the
    input-gradient path of net_backward)."""
    for i in reversed(range(1, len(L))):
        d = f_back(d, L[i][0], inputs[i][0] > 0)
    g = f_back(d, L[0][0])
    return g[0][:, first:], g[1][:, first:]


def _actor_tail(La, ia, s, da, eps, d_lp, scale, B):
    """The tanh, the reparameterisation, the log-prob's own terms and the clamp, back through
    the actor: du = fmaf(da scale, 1 - y y, d_lp (2 y)); dls = in_range ? fmaf(du sigma, eps,
    -d_lp) : 0."""
    y = s["y"]
    t1 = f_mul(da, exact(float(np.float32(scale))))
    om = f_sub(exact(1.0), f_mul(y, y))
    t2 = f_mul((np.broadcast_to(d_lp[0], y[0].shape), np.broadcast_to(d_lp[1], y[0].shape)),
               (2.0 * y[0], 2.0 * y[1]))
    du = f_fma(t1, om, t2)
    eps = np.asarray(eps, np.float64)
    dls = f_fma(f_mul(du, s["sigma"]), exact(eps),
                (np.broadcast_to(-d_lp[0], y[0].shape), np.broadcast_to(d_lp[1], y[0].shape)))
    dls = (np.where(s["in_range"], dls[0], 0.0), np.where(s["in_range"], dls[1], 0.0))
    return backward(La, ia, _cat(du, dls), tile_depth(B))


# ---------------------------------------------------------------- SAC
def sac_critic(La, Lc1, Lc2, Lt1, Lt2, rows, noise, gamma, log_alpha, scale, bias, lo, hi):
    """sac_critic_kernel over sampled windows.  rows: replay_update_reference.gather's (obs,
    actions [B, A], rewards, done, boot_obs) of float32 values; L* [(W, b)] float32 values in
    float64; noise [B, A] (eps').  Returns dict of (value, bar): grads1, grads2, q1, q2,
    returns, sums (2), and ok [B]."""
    obs, act, rewards, done, boot = _rows(rows)
    B = len(obs[0])
    alpha = f_alpha(log_alpha)
    s, _, _ = _squashed_head(La, boot, noise, lo, hi, False)
    xb = _cat(boot, _action(s, scale, bias))
    qt = f_min(_col(forward(Lt1, xb, False)[0], 0), _col(forward(Lt2, xb, False)[0], 0))
    lp = f_sum(s["term"])
    ret = sac_nstep(f_sub(qt, f_mul(alpha, lp)), rewards, done, gamma)
    x = exact(np.concatenate([obs[0], np.asarray(act, np.float64)], axis=1))
    out = {"returns": ret, "ok": np.ones(B, dtype=bool), "grads": [], "sums": []}
    for k, L in (("1", Lc1), ("2", Lc2)):
        q, inputs, ok = forward(L, x, True)
        out["ok"] &= ok
        q = _col(q, 0)
        _, d, sq = _mse_grad(q, ret, B)
        out["q" + k] = q
        out["grads" + k] = backward(L, inputs, (d[0][:, None], d[1][:, None]), tile_depth(B))
        out["sums"].append(sq)
    return out


def sac_actor(La, Lc1, Lc2, obs, noise, log_alpha, scale, bias, lo, hi):
    """sac_actor_kernel over sampled windows: obs [B, F] float32 values, noise [B, A] (eps).
    Returns dict of (value, bar): grads, log_probs, sums (sum min(Q1, Q2), sum log pi), and ok
    [B] (the ReLU masks, the clamp gates and the argmin)."""
    obs = exact(np.asarray(obs, np.float64))
    B, F = obs[0].shape
    alpha = f_alpha(log_alpha)
    s, ia, ok = _squashed_head(La, obs, noise, lo, hi, True)
    ok = ok & s["ok"]
    x = _cat(obs, _action(s, scale, bias))
    q1, i1, k1 = forward(Lc1, x, True)
    q2, i2, k2 = forward(Lc2, x, True)
    q1, q2 = _col(q1, 0), _col(q2, 0)
    ok &= k1 & k2 & (np.abs(q1[0] - q2[0]) > q1[1] + q2[1])
    first = q1[0] <= q2[0]
    lp = f_sum(s["term"])
    Mf = exact(float(B))
    d_q = f_div(exact(-1.0), Mf)
    d_lp = f_div(alpha, Mf)
    da = None
    for L, inputs, pick in ((Lc1, i1, first), (Lc2, i2, ~first)):
        d = (np.where(pick, d_q[0], 0.0)[:, None], np.where(pick, d_q[1], 0.0)[:, None])
        g = input_grad(L, inputs, d, F)
        da = g if da is None else f_add(da, g)
    qmin = (np.where(first, q1[0], q2[0]), np.where(first, q1[1], q2[1]))
    return {"grads": _actor_tail(La, ia, s, da, noise, d_lp, scale, B), "log_probs": lp,
            "sums": [double_sum(qmin, 16), double_sum(lp, 16)], "ok": ok}


# ---------------------------------------------------------------- discrete SAC
def log_softmax(z):
    """The kernels' log pi_c = (z_c - max) - logf(sum_c expf(z_c - max)) and pi_c = expf(log
    pi_c): the max's own error cancels (q_update_bounds._softmax_parts), so log pi is bounded as
    if the exact max were subtracted."""
    mx, e, s = _softmax_parts(z)
    v = z[0] - mx[0][:, None]
    d = (v, _rnd(v, z[1]) + UREL * mx[1][:, None])
    ls = f_log(s)
    lp = f_sub(d, (ls[0][:, None], ls[1][:, None]))
    return lp, f_exp(lp)


def sac_discrete_critic(La, Lq1, Lq2, Lt1, Lt2, rows, gamma, log_alpha):
    """sac_discrete_critic_kernel.  rows: dqn_update_reference.gather's (obs, actions [B],
    rewards, done, boot_obs).  Returns dict of (value, bar): grads1, grads2, q1, q2, returns,
    sums (2), and ok [B]."""
    obs, act, rewards, done, boot = _rows(rows)
    act = act.reshape(-1)
    B = len(act)
    r = np.arange(B)
    alpha = f_alpha(log_alpha)
    lp, pi = log_softmax(forward(La, boot, False)[0])
    m = f_min(forward(Lt1, boot, False)[0], forward(Lt2, boot, False)[0])
    v = f_dot(pi, f_sub(m, f_mul(alpha, lp)))
    ret = nstep(v, rewards, done, gamma)
    out = {"returns": ret, "ok": np.ones(B, dtype=bool), "sums": []}
    for k, L in (("1", Lq1), ("2", Lq2)):
        qs, inputs, ok = forward(L, obs, True)
        out["ok"] &= ok
        q = (qs[0][r, act], qs[1][r, act])
        _, d, sq = _mse_grad(q, ret, B)
        dh = (np.zeros_like(qs[0]), np.zeros_like(qs[0]))
        dh[0][r, act], dh[1][r, act] = d
        out["q" + k] = q
        out["grads" + k] = backward(L, inputs, dh, tile_depth(B))
        out["sums"].append(sq)
    return out


def sac_discrete_actor(La, Lq1, Lq2, obs, log_alpha):
    """sac_discrete_actor_kernel: obs [B, F].  Returns dict of (value, bar): grads, the logit
    deltas [B, A] the kernel back-propagates, entropies,
    sums (sum_g sum_a pi_a min(Q1, Q2)_a, sum_g sum_a pi_a log pi_a), and ok [B]."""
    obs = exact(np.asarray(obs, np.float64))
    B = len(obs[0])
    alpha = f_alpha(log_alpha)
    z, ia, ok = forward(La, obs, True)
    lp, pi = log_softmax(z)
    m = f_min(forward(Lq1, obs, False)[0], forward(Lq2, obs, False)[0])
    h = f_sub(f_mul(alpha, lp), m)
    hbar = f_dot(pi, h)
    pm, plp = f_dot(pi, m), f_dot(pi, lp)
    d = f_mul(f_mul(pi, f_sub(h, (hbar[0][:, None], hbar[1][:, None]))), norm_of(float(B)))
    return {"grads": backward(La, ia, d, tile_depth(B)), "logit_deltas": d,
            "entropies": (-plp[0], plp[1]),
            "sums": [double_sum(pm, 16), double_sum(plp, 16)], "ok": ok}


# ---------------------------------------------------------------- TQC
def _weighted(w, c, u):
    """|tau - 1{u < 0}| times c (clamp(u) or the Huber term, 0 at u = 0) as (value, bar); where
    |u| <= bar either weight may be taken, and the product is continuous."""
    v = w[0] * c[0]
    b = w[0] * c[1] + np.abs(c[0]) * w[1] + w[1] * c[1]
    amb = np.abs(u[0]) <= u[1]
    return v, np.where(amb, np.abs(v) + 1.01 * (np.abs(c[0]) + c[1]), b)


def _fma_sum(t, axis=-1):
    """A fmaf chain sum_k w_k c_k of products given as (value, bar), any order."""
    n = t[0].shape[axis]
    p = np.sum(t[1], axis)
    return np.sum(t[0], axis), _sum_bar(p, np.sum(np.abs(t[0]), axis) + p, n)


def tqc_critic(La, Lc1, Lc2, Lt1, Lt2, rows, noise, gamma, log_alpha, scale, bias, lo, hi, N,
               n_drop):
    """tqc_critic_kernel (two critics).  rows as sac_critic's.  Returns dict of (value, bar):
    grads1, grads2, theta [B, 2, N], returns [B, K] (the kept atoms' returns), q_means,
    target_means [B], sums (sum of the loss rows, sum of q_means), and ok [B]."""
    obs, act, rewards, done, boot = _rows(rows)
    B = len(obs[0])
    K = 2 * (N - n_drop)
    alpha = f_alpha(log_alpha)
    s, _, _ = _squashed_head(La, boot, noise, lo, hi, False)
    xb = _cat(boot, _action(s, scale, bias))
    atoms = _cat(forward(Lt1, xb, False)[0], forward(Lt2, xb, False)[0])       # [B, 2N]
    order = np.argsort(atoms[0], axis=1, kind="stable")[:, :K]
    kept = (np.take_along_axis(atoms[0], order, axis=1),
            np.broadcast_to(atoms[1].max(axis=1, keepdims=True), (B, K)))
    alp = f_mul(alpha, f_sum(s["term"]))
    T = sac_nstep(f_sub(kept, (alp[0][:, None], alp[1][:, None])), rewards, done, gamma)
    x = exact(np.concatenate([obs[0], np.asarray(act, np.float64)], axis=1))
    tv = ((2.0 * np.arange(N) + 1.0) / (2.0 * N)).astype(np.float32).astype(np.float64)
    c_loss = norm_of(float(B) * 2 * N * K)
    out = {"returns": T, "ok": np.ones(B, dtype=bool)}
    thetas, rows_l = [], []
    for k, L in (("1", Lc1), ("2", Lc2)):
        th, inputs, ok = forward(L, x, True)                                   # [B, N]
        out["ok"] &= ok
        thetas.append(th)
        u = f_sub((T[0][:, None, :], T[1][:, None, :]), (th[0][:, :, None], th[1][:, :, None]))
        neg = u[0] < 0
        w = (np.where(neg, 1.0 - tv[None, :, None], tv[None, :, None]),
             np.where(neg, _rnd(1.0 - tv, 0.0)[None, :, None], 0.0))
        au = np.abs(u[0])
        clip = (np.clip(u[0], -1.0, 1.0), np.where((u[0] - u[1] >= 1.0) | (u[0] + u[1] <= -1.0),
                                                   0.0, u[1]))
        hv = np.where(au <= 1.0, 0.5 * u[0] * u[0], au - 0.5)
        hub = _rnd(hv, (np.minimum(au, 1.0) + u[1]) * u[1])
        lsum = _fma_sum(_weighted(w, (hv, hub), u))
        gsum = _fma_sum(_weighted(w, clip, u))
        d = f_mul((-c_loss[0], c_loss[1]), gsum)
        out["grads" + k] = backward(L, inputs, d, tile_depth(B))
        rows_l.append(lsum)
    theta = (np.stack([t[0] for t in thetas], 1), np.stack([t[1] for t in thetas], 1))
    out["theta"] = theta
    flat = (theta[0].reshape(B, -1), theta[1].reshape(B, -1))
    qm = double_mean(flat, 1)
    out["q_means"] = f_round(qm)
    out["target_means"] = f_round(double_mean(T, 1))
    out["sums"] = [double_sum(_cat(*rows_l), 16), double_sum(qm, 16)]
    return out


def tqc_actor(La, Lc1, Lc2, obs, noise, log_alpha, scale, bias, lo, hi, N):
    """tqc_actor_kernel (two critics): obs [B, F], noise [B, A] (eps).  Returns dict of (value,
    bar): grads, log_probs, q_bar [B] (the double mean of all quantiles, as summed), sums (sum
    q_bar, sum log pi), and ok [B]."""
    obs = exact(np.asarray(obs, np.float64))
    B, F = obs[0].shape
    alpha = f_alpha(log_alpha)
    s, ia, ok = _squashed_head(La, obs, noise, lo, hi, True)
    ok = ok & s["ok"]
    x = _cat(obs, _action(s, scale, bias))
    d_q = norm_of(float(B) * 2 * N)
    d = (np.full((B, N), -d_q[0]), np.full((B, N), d_q[1]))
    da, ths = None, []
    for L in (Lc1, Lc2):
        th, inputs, k = forward(L, x, True)
        ok &= k
        ths.append(th)
        g = input_grad(L, inputs, d, F)
        da = g if da is None else f_add(da, g)
    lp = f_sum(s["term"])
    d_lp = f_div(alpha, exact(float(B)))
    qb = double_mean(_cat(*ths), 1)
    return {"grads": _actor_tail(La, ia, s, da, noise, d_lp, scale, B), "log_probs": lp,
            "q_bar": qb, "sums": [double_sum(qb, 16), double_sum(lp, 16)], "ok": ok}

