"""Float64 reference of the action-masked bootstrap of the DQN family (wdb_dqn_update_masked,
wdb_c51_update_masked, include/wdb200.h; algorithms/dqn.py's `boot_mask`).

One rule: a* -- the double-Q argmax, DQN's max_a' and the distributional passes' argmax of the
expectation -- ranges over the valid (non-zero) entries of obs' own mask, the ring's mask row at
the window's slot(n_step); a row with no valid action takes every action.  Everything else is
the unmasked update's.

  * masked_argmax / the *_boot functions: the bootstraps of the four objectives in float64, on
    the float64 networks and helpers of dqn_update_reference, qr_dqn_reference, iqn_reference
    and c51_reference (the torch losses' statement);
  * dqn_masked_pass / c51_masked_pass: q_update_bounds.qr_pass(dqn=True) and c51_pass with the
    masked a*, every output a (value, bar) pair with the same rounding rules and premises (the
    argmax premise compares the first valid maximum with the other valid columns only)."""
import numpy as np

import q_update_bounds as qb
from c51_reference import softmax
from dqn_update_reference import forward
from iqn_reference import embedding, midpoints, parts, trunk_forward
from update_reference import D, exact, f_div, f_mul, f_sub


def boot_mask(ring_mask, windows, n_step):
    """obs' own mask [B, A] of the windows: ring_mask [C, E, Np, A] at slot(n_step)."""
    C, A = ring_mask.shape[0], ring_mask.shape[-1]
    s = (windows[:, 0].astype(np.int64) + n_step) % C
    return ring_mask.reshape(C, -1, A)[s, windows[:, 1].astype(np.int64)]


def valid(mask):
    """The actions a* ranges over: the non-zero entries, or every action of a row with none."""
    v = np.asarray(mask) != 0
    return v | ~v.any(axis=-1, keepdims=True)


def masked_argmax(x, mask):
    """The first maximum of each row of x [B, A] among its valid actions."""
    return np.argmax(np.where(valid(mask), x, -np.inf), axis=1)


# ---------------------------------------------------------------- the torch losses' bootstraps
def dqn_boot(Lq, Lt, boot_obs, mask, double_q):
    """DQN.bootstrap: target(obs')[a*] (double_q) or the max of target(obs') over the valid
    actions [B]."""
    qt = forward(Lt, boot_obs)[0]
    if double_q:
        best = masked_argmax(forward(Lq, boot_obs)[0], mask)
        return qt[np.arange(len(qt)), best]
    return np.where(valid(mask), qt, -np.inf).max(axis=1)


def qr_boot(Lq, Lt, boot_obs, mask, double_q, N):
    """QuantileDQN.bootstrap_quantiles: target(obs')[a*] [B, N], a* over the mean quantile."""
    B = len(boot_obs)
    qt = forward(Lt, boot_obs)[0].reshape(B, -1, N)
    chooser = forward(Lq, boot_obs)[0].reshape(B, -1, N) if double_q else qt
    return qt[np.arange(B), masked_argmax(chooser.mean(axis=2), mask)]


def iqn_boot(models, boot_obs, taus_prime, mask, double_q):
    """ImplicitQuantileDQN.bootstrap_quantiles: the target's Z at tau'_j of a* [B, N'], a* over
    the collapsed head."""
    (Tq, (Wh, bh), Eq), (Tt, (Wth, bth), Et) = parts(models[0]), parts(models[1])
    K = models[0].num_quantile_samples
    psi_t = trunk_forward(Tt, boot_obs)[0]
    if double_q:
        cbar = embedding(Eq, midpoints(K))[0].mean(axis=0)
        chooser = (trunk_forward(Tq, boot_obs)[0] * cbar) @ Wh.T + bh
    else:
        cbar = embedding(Et, midpoints(K))[0].mean(axis=0)
        chooser = (psi_t * cbar) @ Wth.T + bth
    best = masked_argmax(chooser, mask)
    zt = (psi_t[:, None, :] * embedding(Et, taus_prime)[0]) @ Wth.T + bth   # [B, N', A]
    return zt[np.arange(len(boot_obs)), :, best]


def c51_boot(Lq, Lt, boot_obs, mask, double_q, z):
    """CategoricalDQN.bootstrap_distribution: softmax(target.logits(obs')[a*]) [B, N], a* over
    the expectation."""
    B, N = len(boot_obs), len(z)
    lt = forward(Lt, boot_obs)[0].reshape(B, -1, N)
    lc = forward(Lq, boot_obs)[0].reshape(B, -1, N) if double_q else lt
    best = masked_argmax((softmax(lc) * z).sum(axis=2), mask)
    return softmax(lt[np.arange(B), best])


# ---------------------------------------------------------------- the native passes, with bars
def masked_first_argmax(x, mask):
    """q_update_bounds.first_argmax over each row's valid actions: the first valid maximum, and
    whether every other valid column is more than both bars below it."""
    v, b = x
    ok_cols = valid(mask)
    best = masked_argmax(v, mask)
    rows = np.arange(len(v))
    gap = v[rows, best][:, None] - v - b[rows, best][:, None] - b
    gap[rows, best] = np.inf
    gap[~ok_cols] = np.inf
    return best, (gap > 0).all(axis=1)


def dqn_masked_pass(Lq, Lt, rows, mask, gamma, delta, double_q, weights=None):
    """dqn_tile_pass<kWeighted, kMasked = true>: qr_pass(dqn=True) with the masked bootstrap.
    mask [B, A]: obs' own mask rows (boot_mask)."""
    obs, a, rewards, done, boot_obs = qb._rows(rows)
    kappa = qb.f32(delta)
    B = len(a)
    r = np.arange(B)
    qs, inputs, ok = qb.forward(Lq, obs, True)
    qt = qb.forward(Lt, boot_obs, False)[0]
    if double_q:
        best, k = masked_first_argmax(qb.forward(Lq, boot_obs, False)[0], mask)
        ok &= k
        boot = (qt[0][r, best], qt[1][r, best])
    else:                                      # the max over the valid columns: 1-Lipschitz
        best = masked_argmax(qt[0], mask)
        boot = (qt[0][r, best], np.where(valid(mask), qt[1], 0.0).max(axis=1))
    w = None if weights is None else exact(np.asarray(weights, np.float32).astype(np.float64))
    wv = np.ones(B) if weights is None else w[0]
    T = qb.nstep(boot, rewards, done, gamma)
    q = (qs[0][r, a], qs[1][r, a])
    diff = f_sub(q, T)
    c = qb.f_clip(diff, -kappa, kappa)
    if w is not None:
        c = f_mul(c, w)
    dq = f_mul(c, qb.norm_of(float(B)))
    dh = (np.zeros_like(qs[0]), np.zeros_like(qs[0]))
    dh[0][r, a], dh[1][r, a] = dq
    h, hb = qb.huber_terms(diff, kappa)
    sums = [qb.double_sum((h * wv, hb * wv + 2 * D * h * wv), 16),
            qb.double_sum((q[0], q[1]), 16)]
    grads = qb.backward(Lq, inputs, dh, qb.tile_depth(B))
    return {"grads": grads, "q_values": q, "returns": T, "sums": sums, "ok": ok}


def c51_masked_pass(Lq, Lt, rows, mask, gamma, double_q, z, dz, weights=None):
    """c51_tile_pass<kWeighted, kMasked = true>: q_update_bounds.c51_pass with the masked a*."""
    obs, a, rewards, done, boot_obs = qb._rows(rows)
    z = np.asarray(z, np.float32).astype(np.float64)
    dz = qb.f32(dz)
    N = z.size
    B = len(a)
    r = np.arange(B)
    ls, inputs, ok = qb.forward(Lq, obs, True)
    lt = qb.forward(Lt, boot_obs, False)[0]
    lc = qb.forward(Lq, boot_obs, False)[0] if double_q else lt
    A = ls[0].shape[1] // N
    sh = lambda x: (x[0].reshape(B, A, N), x[1].reshape(B, A, N))  # noqa: E731
    lc, lt, ls3 = sh(lc), sh(lt), sh(ls)
    _, e, s = qb._softmax_parts(lc)
    qc = f_div(qb.f_dot(exact(z), e), s)
    best, k = masked_first_argmax(qc, mask)
    ok &= k
    _, e, s = qb._softmax_parts((lt[0][r, best], lt[1][r, best]))
    pb = f_div(e, (s[0][:, None], s[1][:, None]))
    tz = qb.f_clip(qb.nstep(exact(np.broadcast_to(z, (B, N))), rewards, done, gamma),
                   z[0], z[-1])
    diff = f_sub((tz[0][:, None, :], tz[1][:, None, :]), exact(z[None, :, None]))
    c = f_sub(exact(1.0), f_div((np.abs(diff[0]), diff[1]), exact(dz)))
    m = qb.f_dot(qb.f_clip(c, 0.0, 1.0), (pb[0][:, None, :], pb[1][:, None, :]), axis=2)
    sm = qb.f_sum(m)
    rb = (np.sum(z * m[0], 1),
          np.sum(np.abs(z) * m[1], 1) + (N + 2) * D * np.sum(np.abs(z) * (m[0] + m[1]), 1))
    lo = (ls3[0][r, a], ls3[1][r, a])
    mx, e, s = qb._softmax_parts(lo)
    p = f_div(e, (s[0][:, None], s[1][:, None]))
    d = f_sub(f_mul(p, (sm[0][:, None], sm[1][:, None])), m)
    wv = np.ones(B) if weights is None else np.asarray(weights, np.float32).astype(np.float64)
    if weights is not None:
        d = f_mul(d, exact(wv[:, None]))
    d = f_mul(d, qb.norm_of(float(B)))
    dh = (np.zeros((B, A, N)), np.zeros((B, A, N)))
    dh[0][r, a], dh[1][r, a] = d
    dh = (dh[0].reshape(B, A * N), dh[1].reshape(B, A * N))
    lse_v = mx[0] + np.log(s[0])
    lse_b = -np.log1p(-s[1] / s[0]) + 4 * D * (np.abs(mx[0]) + np.abs(np.log(s[0])))
    gap = (lse_v[:, None] - lo[0], lse_b[:, None] + lo[1])
    t = (wv[:, None] * m[0] * gap[0],
         wv[:, None] * (m[0] * gap[1] + m[1] * (np.abs(gap[0]) + gap[1])
                        + 4 * D * np.abs(m[0] * gap[0])))
    qbar = (np.sum(z * p[0], 1),
            np.sum(np.abs(z) * p[1], 1) + (N + 2) * D * np.sum(np.abs(z) * (p[0] + p[1]), 1))
    sums = [qb.double_sum(t, 16 + N), qb.double_sum(qbar, 16)]
    depth = qb.tile_depth(B)
    grads_head = qb.f_grad(dh, inputs[-1], depth)
    grads = []
    if len(Lq) > 1:
        dpsi = qb.f_back(dh, Lq[-1][0], inputs[-1][0] > 0)
        grads = qb.backward(Lq[:-1], inputs[:-1], dpsi, depth)
    return {"grads": grads + list(grads_head), "q_values": qb.f_round(qbar),
            "returns": qb.f_round(rb), "sums": sums, "ok": ok}
