"""Float64 reference with error bars of the DQN-family replay update passes: wdb_dqn_update_sampled
and _prioritized (dqn_pass_kernel), wdb_qr_dqn_update_sampled, wdb_iqn_update_sampled and
wdb_c51_update_sampled (include/wdb200.h), uniform and importance-weighted.

Every output comes as a pair (value, bar): the float64 value of the operation on the kernel's
float32 inputs, and a bound on how far a correct float32 evaluation can lie from it.  The values
are those of dqn_update_reference, per_reference, qr_dqn_reference, iqn_reference and
c51_reference, which stay the statement of the objective; this module adds the bars, carried
through the kernels' float32 operations by update_reference's rules (u = 2**-24, a float32
operation on inputs within P rounds once: P + u/(1+u) (|v| + P); expf within 2 ulp, logf 1 ulp)
and these:
  * a sum of n float32 terms (fmaf chains included) in any order: n u sum|terms| plus the
    propagated input bars; exact (bar 0) when every term is an exact zero;
  * cosf: 2 ulp (|x| < 48039) plus the argument's error |sin x| bar_x + bar_x**2 / 2;
  * fminf / fmaxf / a clip / a max over columns: exact and 1-Lipschitz, so the bar passes
    through, and is 0 where the value is clamped by more than its bar;
  * double accumulations: (terms + 1) 2**-53 sum|terms| on top of the terms' bars;
  * gradient accumulations follow the kernels: layer_grad adds kRows = 16 rows per tile into
    shared memory (`calls` times per tile), over ceil(tiles / grid) tiles per CTA, and
    ddpg_reduce_kernel sums up to 132 CTA partials; a term's path through that tree has at most
    16 + calls * ceil(tiles / grid) + grid roundings.
The inputs are the float32 values the kernel reads: observations, rewards, weights, the support,
float32(delta_z), gamma, kappa / delta and the taus.  What the kernel computes from them -- the
1 / B style normalisers, QR-DQN's and c-bar's midpoint levels, IQN's float(pi c) frequencies --
is charged as a rounding, so the values stay those of the exact formulas.

Branch premises.  Where a decision depends on a computed value the reference requires every
float32 evaluation within the bars to take the value's branch, per row (`ok`):
  * the backward ReLU masks: |z| > bar for the online trunk on obs and IQN's online tau
    embedding (the forwards on obs' and c-bar only use max(z, 0), which is 1-Lipschitz);
  * the bootstrap argmax: the first maximum beats every other column by more than both bars
    (DQN's max target needs none: the max is 1-Lipschitz);
  * the quantile indicator 1{u < 0} of QR-DQN and IQN: |u| > bar.
Huber's clip, C51's target clamp and its projection clip are continuous: bars, no premise.

How tight.  The bars are worst-case running bounds: every sum is charged n u sum|terms|, and a
gradient element's bar adds up its rows' absolute contributions while its value may cancel
across them.  Where gradients are small differences of large terms -- C51's p sum m - m through
two hidden layers -- an element's bar can be several percent of it (the first layer at C51's
run shape); DQN's are about 1e-4 to 1e-3 of each element.  So the bars pin what a norm-wise
check cannot see -- small elements, signs, exact zeros -- but for the large elements of the
deep layers they are looser than a 2e-4 norm-wise test, which the per-pass tests keep."""
import math

import numpy as np

from update_reference import D, TINY, U, UREL, _rnd, exact, f_add, f_div, f_exp, f_mul, f_sub

KROWS = 16
NSM = 132


def gam(n):
    n = np.asarray(n, dtype=np.float64)
    return n * U / (1.0 - n * U)


def _sum_bar(p, mag, n):
    return np.where(mag > 0, p + gam(n) * mag + n * TINY, 0.0)


def f_sum(x, axis=-1):
    """Float32 sum of the terms along axis, any order."""
    n = x[0].shape[axis]
    p = np.sum(x[1], axis)
    return np.sum(x[0], axis), _sum_bar(p, np.sum(np.abs(x[0]), axis) + p, n)


def f_dot(a, b, axis=-1):
    """Float32 sum along axis of the products a * b (fmaf chains), any order."""
    av, ab = np.broadcast_arrays(*a)
    bv, bb = np.broadcast_arrays(*b)
    n = np.broadcast_shapes(av.shape, bv.shape)[axis]
    p = np.sum(np.abs(av) * bb + np.abs(bv) * ab + ab * bb, axis)
    return np.sum(av * bv, axis), _sum_bar(p, np.sum(np.abs(av * bv), axis) + p, n)


def f_linear(x, W, b):
    """x @ W.T + b: layer_forward's fmaf chain over the inputs, then the bias add."""
    v = x[0] @ W.T + b
    p = x[1] @ np.abs(W).T
    return v, _sum_bar(p, np.abs(x[0]) @ np.abs(W).T + np.abs(b) + p, W.shape[1] + 1)


def f_back(d, W, mask=None):
    """d @ W (layer_backward / block_backward), zeroed where mask is False."""
    v = d[0] @ W
    p = d[1] @ np.abs(W)
    b = _sum_bar(p, np.abs(d[0]) @ np.abs(W) + p, W.shape[0])
    if mask is None:
        return v, b
    return np.where(mask, v, 0.0), np.where(mask, b, 0.0)


def f_grad(d, x, depth):
    """(sum_r d_r x_r^T, sum_r d_r) over the leading rows of d [..., out] and x [..., in]."""
    dv, db = (a.reshape(-1, a.shape[-1]) for a in d)
    xv, xb = (a.reshape(-1, a.shape[-1]) for a in x)
    n = depth
    p = np.abs(dv).T @ xb + db.T @ np.abs(xv) + db.T @ xb
    gw = (dv.T @ xv, _sum_bar(p, np.abs(dv).T @ np.abs(xv) + p, n))
    pb = db.sum(axis=0)
    gb = (dv.sum(axis=0), _sum_bar(pb, np.abs(dv).sum(axis=0) + pb, n))
    return gw, gb


def f_clip(x, lo, hi):
    v, b = x
    c = np.clip(v, lo, hi)
    return c, np.where((v - b >= hi) | (v + b <= lo), 0.0, b)


def f_max(x, axis=-1):
    return np.max(x[0], axis), np.max(x[1], axis)


def relu(z, decide):
    """max(z, 0): decide (a backward mask reads it) requires |z| > bar, per leading row."""
    v, b = z
    out = (np.maximum(v, 0.0), np.where(v > 0, b, 0.0) if decide else
           np.where(v + b > 0, b, 0.0))
    if not decide:
        return out, np.ones(len(v), dtype=bool)
    bad = np.abs(v) <= b
    return out, ~bad.reshape(len(v), -1).any(axis=1)


def first_argmax(x):
    """The first maximum of each row of x [B, A], and whether every other column is more than
    both bars below it."""
    v, b = x
    best = np.argmax(v, axis=1)
    rows = np.arange(len(v))
    gap = v[rows, best][:, None] - v - b[rows, best][:, None] - b
    gap[rows, best] = np.inf
    return best, (gap > 0).all(axis=1)


def f_round(x):
    """A double rounded to float32."""
    return x[0], _rnd(x[0], x[1])


def norm_of(den):
    """(float)(1.0 / den) with den a double product of up to three exact factors."""
    v = 1.0 / den
    return v, _rnd(v, 3 * D * v)


def f32(x):
    return np.float64(np.float32(x))


def double_sum(terms, extra=0):
    """Sum of double terms (value, bar) accumulated in double in any order, each term already
    carrying its own double roundings in its bar."""
    v, b = (np.asarray(a, dtype=np.float64).ravel() for a in terms)
    n = v.size + extra
    return math.fsum(v.tolist()), float(np.sum(b)) + (n + 1) * D * float(np.sum(np.abs(v) + b))


def double_mean(x, axis):
    """sum_axis (double) x / n, x float32 values with bars."""
    n = x[0].shape[axis]
    v = np.sum(x[0], axis) / n
    mag = np.sum(np.abs(x[0]) + x[1], axis) / n
    return v, np.sum(x[1], axis) / n + (n + 2) * D * mag


def huber_terms(u, kappa):
    """huber(u, kappa) in double of a float u with its bar: |dh| <= (min(|u|, k) + b) b."""
    v, b = u
    au = np.abs(v)
    h = np.where(au < kappa, 0.5 * au * au, kappa * (au - 0.5 * kappa))
    return h, (np.minimum(au, kappa) + b) * b + 6 * D * h


def tile_depth(B, calls=1):
    tiles = -(-B // KROWS)
    grid = min(tiles, NSM)
    return KROWS + calls * -(-tiles // grid) + grid


def nstep(boot, rewards, done, gamma):
    """DQN's n-step recursion ret = (om * gamma) * ret + r on boot [B, ...]; rewards / done
    [n_step, B] float32."""
    ret = boot
    g = f32(gamma)
    extra = (slice(None),) + (None,) * (boot[0].ndim - 1)
    for j in reversed(range(rewards.shape[0])):
        om = np.where(done[j] != 0, 0.0, g)[extra]
        r = np.asarray(rewards[j], dtype=np.float64)[extra]
        ret = f_add(f_mul(exact(np.broadcast_to(om, ret[0].shape)), ret),
                    exact(np.broadcast_to(r, ret[0].shape)))
    return ret


def forward(L, x, decide):
    """The head output, each layer's input and the per-row premise of the hidden ReLUs."""
    ok = np.ones(len(x[0]), dtype=bool)
    inputs = []
    for i, (W, b) in enumerate(L):
        inputs.append(x)
        z = f_linear(x, W, b)
        if i < len(L) - 1:
            x, k = relu(z, decide)
            ok &= k
        else:
            x = z
    return x, inputs, ok


def trunk(L, x, decide):
    """The hidden Linear + ReLU layers L alone: their output, each layer's input and the
    per-row premise."""
    ok = np.ones(len(x[0]), dtype=bool)
    inputs = []
    for W, b in L:
        inputs.append(x)
        x, k = relu(f_linear(x, W, b), decide)
        ok &= k
    return x, inputs, ok


def backward(L, inputs, d, depth):
    """[dW, db per layer] of the Linear layers L from the delta d at their output."""
    grads = [None] * len(L)
    for i in reversed(range(len(L))):
        grads[i] = f_grad(d, inputs[i], depth)
        if i > 0:
            d = f_back(d, L[i][0], inputs[i][0] > 0)
    return [g for pair in grads for g in pair]


def _rows(rows):
    obs, actions, rewards, done, boot_obs = rows
    return (exact(np.asarray(obs, np.float64)), np.asarray(actions).reshape(-1),
            np.asarray(rewards, np.float64), np.asarray(done), exact(np.asarray(boot_obs, np.float64)))


# ---------------------------------------------------------------- DQN and QR-DQN
def qr_pass(Lq, Lt, rows, gamma, kappa, double_q, N, weights=None, dqn=False):
    """One implementation for both: dqn=True is dqn_pass_kernel (N = 1, the gradient
    clip(Q - R, -delta, delta) w / B, the sums sum w huber and sum Q, the outputs Q and R),
    else qr_dqn_tile_pass.  rows: dqn_update_reference.gather's (obs, actions, rewards, done,
    boot_obs) in float32; Lq, Lt [(W, b)] float32 values in float64.  Returns dict of
    (value, bar): grads, q_values, returns, sums (2), and ok [B] (every premise of the row)."""
    obs, a, rewards, done, boot_obs = _rows(rows)
    kappa = f32(kappa)
    B = len(a)
    r = np.arange(B)
    qs, inputs, ok = forward(Lq, obs, True)
    qt = forward(Lt, boot_obs, False)[0]
    chooser = forward(Lq, boot_obs, False)[0] if double_q else qt
    A = qs[0].shape[1] // N
    w = None if weights is None else exact(np.asarray(weights, np.float32).astype(np.float64))
    wv = np.ones(B) if weights is None else w[0]
    if dqn:
        if double_q:
            best, k = first_argmax(chooser)
            ok &= k
            boot = (qt[0][r, best], qt[1][r, best])
        else:
            boot = f_max(qt)
        T = nstep(boot, rewards, done, gamma)
        q = (qs[0][r, a], qs[1][r, a])
        diff = f_sub(q, T)
        c = f_clip(diff, -kappa, kappa)
        if w is not None:
            c = f_mul(c, w)
        dq = f_mul(c, norm_of(float(B)))
        dh = (np.zeros_like(qs[0]), np.zeros_like(qs[0]))
        dh[0][r, a], dh[1][r, a] = dq
        h, hb = huber_terms(diff, kappa)
        sums = [double_sum((h * wv, hb * wv + 2 * D * h * wv), 16),
                double_sum((q[0], q[1]), 16)]
        out = (q, T)
    else:
        s = f_sum((chooser[0].reshape(B, A, N), chooser[1].reshape(B, A, N)), axis=2)
        best, k = first_argmax(s)
        ok &= k
        qt3 = (qt[0].reshape(B, A, N), qt[1].reshape(B, A, N))
        T = nstep((qt3[0][r, best], qt3[1][r, best]), rewards, done, gamma)
        qs3 = (qs[0].reshape(B, A, N), qs[1].reshape(B, A, N))
        theta = (qs3[0][r, a], qs3[1][r, a])                          # [B, N]
        u = f_sub((T[0][:, None, :], T[1][:, None, :]), (theta[0][:, :, None], theta[1][:, :, None]))
        ok &= (np.abs(u[0]) > u[1]).reshape(B, -1).all(axis=1)
        tv = (2 * np.arange(N) + 1) / (2 * N)
        tau = (tv, _rnd(tv, 0.0))
        m = (np.where(u[0] < 0, 1.0 - tau[0][None, :, None], tau[0][None, :, None]),
             np.where(u[0] < 0, _rnd(1.0 - tau[0], tau[1])[None, :, None], tau[1][None, :, None]))
        acc = f_dot(m, f_clip(u, -kappa, kappa), axis=2)
        if w is not None:
            acc = f_mul(acc, (w[0][:, None], w[1][:, None]))
        dth = f_mul((-acc[0], acc[1]), norm_of(kappa * N * B))
        dh = (np.zeros((B, A, N)), np.zeros((B, A, N)))
        dh[0][r, a], dh[1][r, a] = dth
        dh = (dh[0].reshape(B, A * N), dh[1].reshape(B, A * N))
        h, hb = huber_terms(u, kappa)
        scale = wv[:, None, None] / (kappa * N)
        t = (m[0] * h * scale, (m[0] * hb + m[1] * (h + hb)) * scale + 4 * D * m[0] * h * scale)
        sums = [double_sum(t, 16), double_sum(double_mean(theta, 1), 16)]
        out = (f_round(double_mean(theta, 1)), f_round(double_mean(T, 1)))
    grads = backward(Lq, inputs, dh, tile_depth(B))
    return {"grads": grads, "q_values": out[0], "returns": out[1], "sums": sums, "ok": ok}


# ---------------------------------------------------------------- C51
def _softmax_parts(y):
    """e_j = expf(y_j - max y) and their float sum, of the last axis.  The computed max's own
    error cancels in every use (e / sum e, and max + log(sum e) for the cross-entropy): with
    max' in place of the exact max, each e_j and the sum take one common factor exp(max -
    max').  So e and s are bounded as if the exact max were subtracted; the max's bar only
    widens the magnitude the subtraction rounds."""
    mx = f_max(y)
    v = y[0] - mx[0][..., None]
    e = f_exp((v, _rnd(v, y[1]) + UREL * mx[1][..., None]))
    return mx, e, f_sum(e)


def c51_pass(Lq, Lt, rows, gamma, double_q, z, dz, weights=None):
    """c51_tile_pass.  z: the support (float32 values), dz: float32(delta_z)."""
    obs, a, rewards, done, boot_obs = _rows(rows)
    z = np.asarray(z, np.float32).astype(np.float64)
    dz = f32(dz)
    N = z.size
    B = len(a)
    r = np.arange(B)
    ls, inputs, ok = forward(Lq, obs, True)
    lt = forward(Lt, boot_obs, False)[0]
    lc = forward(Lq, boot_obs, False)[0] if double_q else lt
    A = ls[0].shape[1] // N
    sh = lambda x: (x[0].reshape(B, A, N), x[1].reshape(B, A, N))  # noqa: E731
    lc, lt, ls3 = sh(lc), sh(lt), sh(ls)
    _, e, s = _softmax_parts(lc)
    qc = f_div(f_dot(exact(z), e), s)
    best, k = first_argmax(qc)
    ok &= k
    _, e, s = _softmax_parts((lt[0][r, best], lt[1][r, best]))
    pb = f_div(e, (s[0][:, None], s[1][:, None]))
    tz = f_clip(nstep(exact(np.broadcast_to(z, (B, N))), rewards, done,
                      gamma), z[0], z[-1])
    diff = f_sub((tz[0][:, None, :], tz[1][:, None, :]), exact(z[None, :, None]))
    c = f_sub(exact(1.0), f_div((np.abs(diff[0]), diff[1]), exact(dz)))
    m = f_dot(f_clip(c, 0.0, 1.0), (pb[0][:, None, :], pb[1][:, None, :]), axis=2)   # [B, N]
    sm = f_sum(m)
    rb = (np.sum(z * m[0], 1), np.sum(np.abs(z) * m[1], 1) + (N + 2) * D * np.sum(np.abs(z) * (m[0] + m[1]), 1))
    lo = (ls3[0][r, a], ls3[1][r, a])
    mx, e, s = _softmax_parts(lo)
    p = f_div(e, (s[0][:, None], s[1][:, None]))
    d = f_sub(f_mul(p, (sm[0][:, None], sm[1][:, None])), m)
    wv = np.ones(B) if weights is None else np.asarray(weights, np.float32).astype(np.float64)
    if weights is not None:
        d = f_mul(d, exact(wv[:, None]))
    d = f_mul(d, norm_of(float(B)))
    dh = (np.zeros((B, A, N)), np.zeros((B, A, N)))
    dh[0][r, a], dh[1][r, a] = d
    dh = (dh[0].reshape(B, A * N), dh[1].reshape(B, A * N))
    # the cross-entropy in double: lse = mx + log(s) (the max's error cancels, _softmax_parts)
    lse_v = mx[0] + np.log(s[0])
    lse_b = -np.log1p(-s[1] / s[0]) + 4 * D * (np.abs(mx[0]) + np.abs(np.log(s[0])))
    gap = (lse_v[:, None] - lo[0], lse_b[:, None] + lo[1])
    t = (wv[:, None] * m[0] * gap[0],
         wv[:, None] * (m[0] * gap[1] + m[1] * (np.abs(gap[0]) + gap[1])
                        + 4 * D * np.abs(m[0] * gap[0])))
    qbar = (np.sum(z * p[0], 1), np.sum(np.abs(z) * p[1], 1) + (N + 2) * D * np.sum(np.abs(z) * (p[0] + p[1]), 1))
    sums = [double_sum(t, 16 + N), double_sum(qbar, 16)]
    depth = tile_depth(B)
    L = len(Lq)
    (Wh, bh) = Lq[-1]
    grads_head = f_grad(dh, inputs[-1], depth)
    grads = []
    if L > 1:
        dpsi = f_back(dh, Wh, inputs[-1][0] > 0)
        grads = backward(Lq[:-1], inputs[:-1], dpsi, depth)
    return {"grads": grads + list(grads_head), "q_values": f_round(qbar), "returns": f_round(rb),
            "sums": sums, "ok": ok}


# ---------------------------------------------------------------- IQN
def cos_features(tau, n_cos):
    """cosf(float(tau * float(pi c))): the frequencies' rounding charged."""
    c = np.arange(n_cos)
    fx = np.pi * c
    fe = np.abs(np.float32(fx).astype(np.float64) - fx)
    tv, tb = tau[0][..., None], tau[1][..., None]
    arg_v = tv * fx
    arg = (arg_v, _rnd(arg_v, np.abs(tv) * fe + fx * tb + tb * fe))
    v = np.cos(arg[0])
    b = np.abs(np.sin(arg[0])) * arg[1] + 0.5 * arg[1] ** 2
    return v, b + 2 * (2 * U * (np.abs(v) + b)) + 2 * 2.0 ** -149


def iqn_pass(trunk_q, head_q, emb_q, trunk_t, head_t, emb_t, rows, gamma, kappa, double_q,
             taus, N, K, weights=None):
    """iqn_tile_pass.  trunk_* [(W, b)], head_* / emb_* (W, b); taus float32 [B, N + N']."""
    obs, a, rewards, done, boot_obs = _rows(rows)
    kappa = f32(kappa)
    B = len(a)
    r = np.arange(B)
    taus = np.asarray(taus, np.float32).astype(np.float64)
    n_cos = emb_q[0].shape[1]
    NP = taus.shape[1] - N
    psi, inputs, ok = trunk(trunk_q, obs, True)
    psi_t = trunk(trunk_t, boot_obs, False)[0]

    def cbar(emb):
        tv = (2 * np.arange(K) + 1) / (2 * K)
        cf = cos_features((tv, _rnd(tv, 0.0)), n_cos)
        phi = relu(f_linear(cf, *emb), False)[0]
        return f_div(f_sum((phi[0].T, phi[1].T)), exact(float(K)))

    if double_q:
        psib = trunk(trunk_q, boot_obs, False)[0]
        cb, hc = cbar(emb_q), head_q
    else:
        psib, cb, hc = psi_t, cbar(emb_t), head_t
    chooser = f_linear(f_mul(psib, (cb[0][None], cb[1][None])), *hc)
    best, k = first_argmax(chooser)
    ok &= k
    tp = exact(taus[:, N:])
    phi_t = relu(f_linear(cos_features(tp, n_cos), *emb_t), False)[0]     # [B, N', H]
    zt = f_linear(f_mul((psi_t[0][:, None], psi_t[1][:, None]), phi_t), *head_t)
    T = nstep((zt[0][r, :, best], zt[1][r, :, best]), rewards, done, gamma)
    tq = exact(taus[:, :N])
    cf = cos_features(tq, n_cos)                                           # [B, N, n_cos]
    phi, k = relu(f_linear(cf, *emb_q), True)
    ok &= k
    mg = f_mul((psi[0][:, None], psi[1][:, None]), phi)
    zq = f_linear(mg, *head_q)
    theta = (zq[0][r, :, a], zq[1][r, :, a])                               # [B, N]
    u = f_sub((T[0][:, None, :], T[1][:, None, :]), (theta[0][:, :, None], theta[1][:, :, None]))
    ok &= (np.abs(u[0]) > u[1]).reshape(B, -1).all(axis=1)
    tv = taus[:, :N, None]
    m = (np.where(u[0] < 0, 1.0 - tv, tv), np.where(u[0] < 0, _rnd(1.0 - tv, 0.0), 0.0))
    acc = f_dot(m, f_clip(u, -kappa, kappa), axis=2)
    wv = np.ones(B) if weights is None else np.asarray(weights, np.float32).astype(np.float64)
    if weights is not None:
        acc = f_mul(acc, exact(wv[:, None]))
    dth = f_mul((-acc[0], acc[1]), norm_of(kappa * NP * B))
    A = zq[0].shape[2]
    dz = (np.zeros((B, N, A)), np.zeros((B, N, A)))
    dz[0][r, :, a], dz[1][r, :, a] = dth
    depth_n = tile_depth(B, calls=N)
    head = f_grad(dz, mg, depth_n)
    dmg = f_back(dz, head_q[0])                                            # [B, N, H]
    dpsi = f_dot(dmg, phi, axis=1)                                         # [B, H]
    dphi = f_mul(dmg, (psi[0][:, None], psi[1][:, None]))
    live = phi[0] > 0
    dphi = (np.where(live, dphi[0], 0.0), np.where(live, dphi[1], 0.0))
    emb = f_grad(dphi, cf, depth_n)
    dpsi = (np.where(psi[0] > 0, dpsi[0], 0.0), np.where(psi[0] > 0, dpsi[1], 0.0))
    grads = backward(trunk_q, inputs, dpsi, tile_depth(B))
    h, hb = huber_terms(u, kappa)
    scale = wv[:, None, None] / (kappa * NP)
    t = (m[0] * h * scale, (m[0] * hb + m[1] * (h + hb)) * scale + 4 * D * m[0] * h * scale)
    qbar = double_mean(theta, 1)
    return {"grads": grads + list(head) + list(emb), "q_values": f_round(qbar),
            "returns": f_round(double_mean(T, 1)),
            "sums": [double_sum(t, 16), double_sum(qbar, 16)], "ok": ok}


# ---------------------------------------------------------------- dueling fold and unfold
def centred(x, A, N):
    """x[a N + j] - float(float(sum_c x[c N + j]) / A) of float32 rows x [A N, ...] (exact
    inputs), the sum over c = 0 .. A - 1 (wdb_dueling.cu's centered)."""
    y = np.asarray(x, np.float64).reshape(A, N, -1)
    mean = f_div(f_sum((np.moveaxis(y, 0, -1), np.zeros(y.shape[1:] + (A,)))), exact(float(A)))
    c = f_sub(exact(y), (mean[0][None], mean[1][None]))
    return c[0].reshape(np.shape(x)), c[1].reshape(np.shape(x))


def fold(p, A, N, S):
    """wdb_dueling_fold of the stream parameters p (dueling_reference.stream_params of a float32
    head): [(weight, bias)] of the folded layers as (value, bar) pairs, [hidden (S > 0),]
    output.  Copies are exact; a centred row rounds its sum, its divide and its subtract, and
    S = 0 adds the value row once more."""
    tile = lambda x, reps: exact(np.tile(x, reps))  # noqa: E731
    b = f_add(tile(p["value_ob"], A), centred(p["adv_ob"], A, N))
    ca = centred(p["adv_ow"], A, N)
    if S == 0:
        return [(f_add(tile(p["value_ow"], (A, 1)), ca), b)]
    hidden = (exact(np.concatenate([p["value_hw"], p["adv_hw"]])),
              exact(np.concatenate([p["value_hb"], p["adv_hb"]])))
    vo = tile(p["value_ow"], (A, 1))
    return [hidden, ((np.concatenate([vo[0], ca[0]], axis=1),
                      np.concatenate([vo[1], ca[1]], axis=1)), b)]


def unfold(grads, A, N, S):
    """wdb_dueling_unfold_grads of the folded layers' float32 gradients [(gw, gb)]: the stream
    gradients (dueling_reference.unfold's names) as (value, bar) pairs.  The value rows are
    float32 sums over the A actions in order, the advantage rows centred, the hidden rows
    copies."""
    g = [(np.asarray(w, np.float64), np.asarray(b, np.float64)) for w, b in grads]
    out = {}
    if S > 0:
        (ghw, ghb), (gow, gob) = g
        out["value_hw"], out["adv_hw"] = exact(ghw[:S]), exact(ghw[S:])
        out["value_hb"], out["adv_hb"] = exact(ghb[:S]), exact(ghb[S:])
        gv, ga = gow[:, :S], gow[:, S:]
    else:
        (gow, gob), = g
        gv = ga = gow
    over_a = lambda x: f_sum(exact(np.moveaxis(x.reshape(A, N, -1), 0, -1)))  # noqa: E731
    vo = over_a(gv)
    out["value_ow"] = vo
    vb = over_a(gob)
    out["value_ob"] = (vb[0][:, 0], vb[1][:, 0])
    out["adv_ow"] = centred(ga, A, N)
    out["adv_ob"] = centred(gob, A, N)
    return out
