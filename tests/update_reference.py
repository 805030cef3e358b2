"""Float64 reference of the fused update kernels (csrc/wdb_update.cu), in plain numpy.

It restates, independently of the CUDA code, every entry point of the training update:
  * pg_loss: bootstrapped returns, advantages, the Categorical log-prob / entropy of every head
    (torch.distributions semantics: q = p / sum(p), log(clamp(q, eps32, 1 - eps32)) with
    eps32 = 2**-23, clamp gradients passed for eps32 <= q <= 1 - eps32, both ends inclusive),
    the four loss sums and the gradients of
        loss = mean(-logp * adv) + vf * mean((V - R)^2) - c * sum_k mean(H_k)
    with respect to every head's probabilities and the values.  PPO's clipped surrogate has
    the same gradient at ratio 1, and its policy loss is -mean(adv) = -sums[3] / M;
  * heads_softmax and its backward, dz_j = p_j (g_j - sum_k g_k p_k); a head passed as NULL
    gets zero gradient, the value column is a copy, the padding columns are +0.0;
  * relu_backward_bias: dh * (h > 0) (so -0.0 and NaN mask) and the per-CTA column sums over
    the row partition wdb_relu_backward_bias_rows(rows) defines (passed in as `per`);
  * pad_rows, grad_sumsq (adds to *out) and Adam with clipping in the kernel's own formula:
    float32 betas / eps / lr as the ABI carries them, bias corrections 1 - powf(beta, step).

Error bounds.  Every float output comes as a pair (value, bar): the float64 value of the
operation on the kernel's float32 inputs, and a bound on how far a correct float32 evaluation
may lie from it.  The bar is a running error bound carried through the same sequence of
float32 operations the kernel performs, with u = 2**-24:
  * a float32 operation on inputs known to within P rounds once: bar = P + u/(1+u) (|v| + P)
    (+ 2**-150 in the subnormal range), and 0 when P = 0 and the exact result is a float;
  * propagation is first order plus the cross term: x*y gives |x| by + |y| bx + bx by,
    x/y gives (bx + |x/y| by) / (|y| - by), sqrt(x) gives bx / (sqrt(x) + sqrt(x - bx));
  * the library builds without fast-math: logf is within 1 ulp (<= 2u |result|), expf within
    2 ulp, division and sqrtf are IEEE.  A sequential float32 sum of n terms therefore carries
    at most n roundings of at most its partial sums, i.e. the familiar
    n_roundings * 2**-24 * sum(|terms|); a product of k rounded factors k roundings of |v|.
  * an FMA rounds once where the rule charges the product and the sum separately, so whether
    nvcc contracts `r + gamma * ret`, `ent -= lq * q` or `S += gq * q` does not matter.
What that amounts to, per output (n = head width):
  * returns: R_t = r_t + gamma R_{t+1}: bar_t = gamma bar_{t+1} + 2u (|r_t| + gamma |R_{t+1}|)
    (two roundings per step; the error of later steps decays with gamma <= 1); exact at the
    start of each segment (the bootstrap V or the reward of a done step);
  * adv = R - V: bar_R + u |R - V|; grad_values = 2 vf (V - R) / M: three more roundings;
  * q = p * (1 / z): z a sequential sum of n non-negative terms: about (n + 1) u |q|;
    log q: (n + 1) u + 2u |log q|; the -adv / q term: (bar_adv + (n + 2) u |adv|) / q;
    grad_probs: ((gq - S) / M) / z with S a sequential sum: (n + 4 + ...) u times the
    magnitude |gq| + sum |gq_i q_i|, over M z;
  * softmax: e_j = expf(x_j - max): (|x_j - max| + 4) u relative; p = e / sum e: the sum's n
    roundings and two more;  backward: (n + 2) u p_j (|g_j| + sum_k |g_k p_k|);
  * sums (double): every term's float32 bar, plus (terms + 1) 2**-53 sum |terms| for the
    double accumulation in any order (atomics included);
  * relu bias partials: (rows - 1) u / (1 - (rows - 1) u) * sum |terms| for any summation
    order over the CTA's rows;
  * bit-exact (bar 0): masked dh, pad_rows, the softmax value column and padding columns,
    NULL heads, and the sumsq terms (a float squared in double is exact; only the double sum
    rounds).
Where a decision depends on a computed value (the clamp test of q), the reference requires
every float32 value within the bar to take the same branch as the exact q (`ClampPremise`):
rows that sit exactly on eps or 1 - eps must be built so that z is exact (float32 rows that
sum to 1 in every order), and no other q may lie within its bar of a boundary.
"""
import math

import numpy as np

U = 2.0 ** -24
UREL = U / (1.0 + U)
EPS32 = 2.0 ** -23                    # torch.finfo(torch.float32).eps
SUBNORMAL = 2.0 ** -126
TINY = 2.0 ** -150                    # half the smallest subnormal: RN's absolute error there
D = 2.0 ** -53


# ---------------------------------------------------------------- running error bounds
def exact(v):
    v = np.asarray(v, dtype=np.float64)
    return v, np.zeros_like(v)


def _rnd(v, p):
    """Bar of a float32 result whose exact value from the computed inputs is within p of v."""
    v = np.asarray(v, dtype=np.float64)
    p = np.broadcast_to(np.asarray(p, dtype=np.float64), v.shape)
    mag = np.abs(v) + p
    b = p + UREL * mag + np.where(mag < SUBNORMAL, TINY, 0.0)
    with np.errstate(over="ignore", invalid="ignore"):
        representable = v.astype(np.float32).astype(np.float64) == v
    return np.where((p == 0) & representable, 0.0, b)


def f_add(x, y):
    v = x[0] + y[0]
    return v, _rnd(v, x[1] + y[1])


def f_sub(x, y):
    v = x[0] - y[0]
    return v, _rnd(v, x[1] + y[1])


def f_neg(x):
    return -x[0], x[1]


def f_mul(x, y):
    v = x[0] * y[0]
    return v, _rnd(v, np.abs(x[0]) * y[1] + np.abs(y[0]) * x[1] + x[1] * y[1])


def f_div(x, y):
    v = x[0] / y[0]
    room = np.abs(y[0]) - y[1]
    assert np.all(room > 0), "divisor not bounded away from 0"
    return v, _rnd(v, (x[1] + np.abs(v) * y[1]) / room)


def f_sqrt(x):
    v = np.sqrt(x[0])
    lo = np.sqrt(np.maximum(x[0] - x[1], 0.0))
    with np.errstate(invalid="ignore", divide="ignore"):
        p = np.where(x[1] > 0, x[1] / (v + lo), 0.0)
    return v, _rnd(v, p)


def f_log(x, ulps=1):
    assert np.all(x[0] > x[1])
    v = np.log(x[0])
    p = -np.log1p(-x[1] / x[0])
    return v, p + 2.0 * U * ulps * (np.abs(v) + p)


def f_exp(x, ulps=2):
    v = np.exp(x[0])
    p = v * np.expm1(x[1])
    return v, p + 2.0 * U * ulps * (v + p) + ulps * 2.0 ** -149


def select(cond, x, y):
    return np.where(cond, x[0], y[0]), np.where(cond, x[1], y[1])


def within(kernel, ref, slack=1.0):
    """Worst excess of |kernel - value| over the bar (<= 0 passes) and where it happens."""
    v, b = ref
    k = np.asarray(kernel, dtype=np.float64)
    err = np.abs(k - v) - slack * b
    err = np.where(np.isnan(k) | np.isnan(err), np.inf, err)
    i = int(np.argmax(err)) if err.size else 0
    return (float(err.flat[i]) if err.size else -1.0), i


def sum_double(terms):
    """Sum of float32 terms accumulated in double in any order: value, bar (the terms' own bars
    plus (n + 1) * 2**-53 * sum |terms| for the double additions and this sum's own)."""
    v, b = terms
    n = v.size
    absum = float(np.sum(np.abs(v) + b))
    return math.fsum(v.ravel().tolist()), float(np.sum(b)) + (n + 1) * D * absum


# ---------------------------------------------------------------- pg_loss
class ClampPremise(AssertionError):
    """A q within its bar of the clamp boundary: the branch the kernel takes is not decided."""


def _f32_ceil(x):
    f = x.astype(np.float32)
    return np.where(f.astype(np.float64) < x, np.nextafter(f, np.float32(np.inf)), f)


def _f32_floor(x):
    f = x.astype(np.float32)
    return np.where(f.astype(np.float64) > x, np.nextafter(f, np.float32(-np.inf)), f)


def _inside(q):
    return (q >= EPS32) & (q <= 1.0 - EPS32)


def returns_and_advantages(values, rewards, done, gamma):
    """values / rewards [T, E, Np] float32, done [T, E] int (> 0 = done), gamma a float32.
    -> (returns, advantages) as (value, bar) pairs [T, E, Np]."""
    T = rewards.shape[0]
    v64 = values.astype(np.float64)
    r64 = rewards.astype(np.float64)
    d = np.broadcast_to((done > 0)[:, :, None], rewards.shape)
    g = exact(np.float64(np.float32(gamma)))
    ret_v, ret_b = np.empty_like(r64), np.empty_like(r64)
    ret_v[T - 1] = np.where(d[T - 1], r64[T - 1], v64[T - 1])
    ret_b[T - 1] = 0.0
    for t in range(T - 2, -1, -1):
        s = f_add(exact(r64[t]), f_mul(g, (ret_v[t + 1], ret_b[t + 1])))
        ret_v[t] = np.where(d[t], r64[t], s[0])
        ret_b[t] = np.where(d[t], 0.0, s[1])
    ret = (ret_v, ret_b)
    return ret, f_sub(ret, exact(v64))


def pg_loss(probs, values, actions, rewards, done, gamma, vf_coeff, entropy_coeff):
    """The outputs of wdb_pg_loss_and_grads on these float32 inputs.
    probs: list of [T, E, Np, A_k] float32 (unnormalised rows and zeros allowed), actions
    [T, E, Np, n_heads] int, the coefficients as the float32 values the ABI carries.
    Returns dict: returns, adv, grad_values, grad_probs (list), sums (4 x (value, bar): sum
    -logp*adv, sum (V-R)^2, sum_k sum H_k, sum adv)."""
    T, E, Np = rewards.shape
    M = float(T) * E * Np
    vf = np.float64(np.float32(vf_coeff))
    c = exact(np.float64(np.float32(entropy_coeff)))
    ret, adv = returns_and_advantages(values, rewards, done, gamma)
    dv = f_neg(adv)                                    # v - ret is -(ret - v), bit for bit
    inv_m = (1.0 / M, _rnd(1.0 / M, D / M))            # (float)(1.0 / M)
    grad_values = f_mul(f_mul(exact(2.0 * vf), dv), inv_m)
    logp = exact(np.zeros((T, E, Np)))
    grad_probs, ent_terms = [], []
    for k, pk in enumerate(probs):
        P = pk.astype(np.float64)
        A = P.shape[-1]
        a = actions[..., k]
        z = exact(np.zeros((T, E, Np)))
        for j in range(A):
            z = f_add(z, exact(P[..., j]))
        inv_z = f_div(exact(np.ones_like(z[0])), z)
        ent = exact(np.zeros((T, E, Np)))
        S = exact(np.zeros((T, E, Np)))
        lq_a = exact(np.zeros((T, E, Np)))
        gq_v, gq_b = np.empty_like(P), np.empty_like(P)
        for j in range(A):
            q = f_mul(exact(P[..., j]), inv_z)
            inside = _inside(q[0])
            if not (np.array_equal(_inside(_f32_ceil(q[0] - q[1])), inside)
                    and np.array_equal(_inside(_f32_floor(q[0] + q[1])), inside)):
                raise ClampPremise(f"head {k} column {j}: q within its bar of the clamp")
            # a clamped q is eps or 1 - eps exactly on both sides
            qc = (np.clip(q[0], EPS32, 1.0 - EPS32), np.where(inside, q[1], 0.0))
            lq = f_log(qc)
            ent = f_sub(ent, f_mul(lq, q))
            gq = f_mul(c, f_add(lq, exact(inside.astype(np.float64))))
            taken = a == j
            with np.errstate(divide="ignore", invalid="ignore"):
                q_safe = (np.where(inside, q[0], 1.0), np.where(inside, q[1], 0.0))
                gq = select(taken & inside, f_sub(gq, f_div(adv, q_safe)), gq)
            lq_a = select(taken, lq, lq_a)
            S = f_add(S, f_mul(gq, q))
            gq_v[..., j], gq_b[..., j] = gq
        logp = f_add(logp, lq_a)
        ent_terms.append(ent)
        gp = f_mul(f_mul(f_sub((gq_v, gq_b), (S[0][..., None], S[1][..., None])), inv_m),
                   (inv_z[0][..., None], inv_z[1][..., None]))
        grad_probs.append(gp)
    pol = f_mul(f_neg(logp), adv)
    sq = (dv[0] ** 2, 2.0 * np.abs(dv[0]) * dv[1] + dv[1] ** 2)
    ent_all = (np.stack([e[0] for e in ent_terms]), np.stack([e[1] for e in ent_terms]))
    sums = [sum_double(pol), sum_double(sq), sum_double(ent_all), sum_double(adv)]
    return dict(returns=ret, adv=adv, grad_values=grad_values, grad_probs=grad_probs,
                sums=sums, M=M)


def pg_loss_value(sums, M, vf_coeff, entropy_coeff, ppo=False):
    """fused_pg_loss's loss: (policy + vf * vf_sum - c * ent) / M in double, then float32."""
    (s0, b0), (s1, b1), (s2, b2), (s3, b3) = sums
    pol, bp = (-s3, b3) if ppo else (s0, b0)
    v = (pol + vf_coeff * s1 - entropy_coeff * s2) / M
    mag = (abs(pol) + bp + abs(vf_coeff) * (abs(s1) + b1) + abs(entropy_coeff) * (abs(s2) + b2)) / M
    bar = (bp + abs(vf_coeff) * b1 + abs(entropy_coeff) * b2) / M + 8 * D * mag
    return v, bar + UREL * (abs(v) + bar) + TINY


# ---------------------------------------------------------------- heads softmax
def heads_softmax(logits, A0, A1):
    """logits [rows, pitch] float32 -> (p0, p1 or None) as (value, bar) pairs and the value
    column (a float32 copy)."""
    x = logits.astype(np.float64)
    out = []
    for off, n in ((0, A0), (A0, A1)):
        if n == 0:
            out.append(None)
            continue
        h = x[:, off:off + n]
        mx = h.max(axis=1)
        es = [f_exp(f_sub(exact(h[:, j]), exact(mx))) for j in range(n)]
        s = exact(np.zeros(len(x)))
        for e in es:
            s = f_add(s, e)
        inv = f_div(exact(np.ones(len(x))), s)
        ps = [f_mul(e, inv) for e in es]
        out.append((np.stack([p[0] for p in ps], 1), np.stack([p[1] for p in ps], 1)))
    return out[0], out[1], logits[:, A0 + A1].copy()


def heads_softmax_backward(p0, p1, g0, g1, gv, A0, A1, pitch):
    """float32 arrays (g0 / g1 / gv may be None) -> dz [rows, pitch] as (value, bar); bar 0
    (bit-exact) on NULL heads, the value column and the padding columns (+0.0)."""
    rows = len(p0)
    dz_v, dz_b = np.zeros((rows, pitch)), np.zeros((rows, pitch))
    for off, n, p, g in ((0, A0, p0, g0), (A0, A1, p1, g1)):
        if n == 0 or g is None:
            continue
        P, G = p.astype(np.float64), g.astype(np.float64)
        dot = exact(np.zeros(rows))
        for j in range(n):
            dot = f_add(dot, f_mul(exact(G[:, j]), exact(P[:, j])))
        for j in range(n):
            dz_v[:, off + j], dz_b[:, off + j] = f_mul(exact(P[:, j]), f_sub(exact(G[:, j]), dot))
    if gv is not None:
        dz_v[:, A0 + A1] = gv
    return dz_v, dz_b


# ---------------------------------------------------------------- relu backward, pad, sumsq
def relu_backward_bias(dh, h, per):
    """-> masked dh (float32, bit-exact) and the [ceil(rows / per), width] partial column sums
    as (value, bar)."""
    masked = np.where(h > 0, dh, np.float32(0.0)).astype(np.float32)
    rows = len(dh)
    starts = np.arange(0, rows, per)
    m64 = masked.astype(np.float64)
    v = np.add.reduceat(m64, starts, axis=0)
    a = np.add.reduceat(np.abs(m64), starts, axis=0)
    n = np.minimum(per, rows - starts)[:, None].astype(np.float64)
    k = np.maximum(n - 1, 0)
    return masked, (v, (k * U / (1.0 - k * U) + n * D) * a)


def pad_rows(src, pitch):
    out = np.zeros((len(src), pitch), dtype=np.float32)
    out[:, :src.shape[1]] = src
    return out


def grad_sumsq(g, out0):
    """*out + sum g^2: each square exact in double; (value, bar) for the double sum."""
    sq = g.astype(np.float64).ravel() ** 2
    chunks = np.array_split(sq, max(1, sq.size // 1_000_000))
    v = math.fsum([float(out0)] + [math.fsum(c.tolist()) for c in chunks])
    return v, (sq.size + 2) * D * (abs(float(out0)) + float(np.sum(sq)))


# ---------------------------------------------------------------- Adam
def powf_bar(beta, step):
    """Host powf(beta, step): within 1 ulp, exact for step 1 (the power is the float itself)."""
    v = float(beta) ** step
    return v, (0.0 if step == 1 else 2.0 * U * v)


def adam_step(p, g, m, v, lr, beta1, beta2, eps, step, max_norm=0.0, sumsq=None):
    """wdb_adam_step on float32 arrays; sumsq the double the clip factor is read from.
    Returns dict of (value, bar): params, grads (the scaled gradient written back), exp_avg,
    exp_avg_sq."""
    f = lambda x: np.float64(np.float32(x))            # noqa: E731  the ABI's float32 values
    lr, b1, b2, eps, max_norm = f(lr), f(beta1), f(beta2), f(eps), f(max_norm)
    P, G, Mm, V = (exact(x.astype(np.float64)) for x in (p, g, m, v))
    if max_norm > 0:
        s = float(sumsq)
        norm = (math.sqrt(s), _rnd(math.sqrt(s), D * math.sqrt(s)))      # (float)sqrt(double)
        ratio = f_div(exact(max_norm), f_add(norm, exact(f(1.0e-6))))
        r, rb = float(ratio[0]), float(ratio[1])
        clip = (min(1.0, r), 0.0 if r - rb >= 1.0 else rb)
    else:
        clip = (1.0, 0.0)
    gi = f_mul(G, (np.float64(clip[0]), np.float64(clip[1])))
    mi = f_add(f_mul(exact(b1), Mm), f_mul(f_sub(exact(1.0), exact(b1)), gi))
    vi = f_add(f_mul(exact(b2), V), f_mul(f_mul(f_sub(exact(1.0), exact(b2)), gi), gi))
    bias1 = f_sub(exact(1.0), powf_bar(b1, step))
    bias2_sqrt = f_sqrt(f_sub(exact(1.0), powf_bar(b2, step)))
    denom = f_add(f_div(f_sqrt(vi), (np.float64(bias2_sqrt[0]), np.float64(bias2_sqrt[1]))),
                  exact(eps))
    upd = f_mul(f_div(exact(lr), (np.float64(bias1[0]), np.float64(bias1[1]))), f_div(mi, denom))
    return dict(params=f_sub(P, upd), grads=gi, exp_avg=mi, exp_avg_sq=vi, update=upd,
                clip=clip, denom=denom)


def adam_torch_deviation(ref, g, m, v, lr, beta1, beta2, eps, step, clipped_n=0):
    """Bound on |torch.optim.Adam (+ clip_grad_norm_) - this reference| for one step from the
    same state, on top of the float32 bars.  torch takes the betas as Python doubles (bias
    corrections 1 - beta**step in double, 1 - beta cast to float32 for the moment updates),
    the kernel their float32 values; clip_grad_norm_ computes the norm in float32 (relative
    error <= (n + 2) u over n elements).  First order in each perturbation:
      dm <= |b1_f - b1| |m| + |w1_t - w1_k| |g| + w1 |g| eps_g
      dv <= |b2_f - b2| v + |w2_t - w2_k| g^2 + 2 w2 g^2 eps_g
      dupd <= lr / bias1 * dm / denom + |upd| (dbias1 / bias1 + (dv / v + dbias2 / bias2) / 2)."""
    f = lambda x: float(np.float32(x))                 # noqa: E731
    b1f, b2f = f(beta1), f(beta2)
    w1t, w2t = f(1.0 - beta1), f(1.0 - beta2)
    w1k, w2k = 1.0 - b1f, 1.0 - b2f
    g, m, v = (x.astype(np.float64) for x in (g, m, v))
    eg = (clipped_n + 2) * U if clipped_n else 0.0
    gi = np.abs(g) * ref["clip"][0]
    dm = abs(b1f - beta1) * np.abs(m) + abs(w1t - w1k) * gi + w1k * gi * eg
    dv = abs(b2f - beta2) * v + abs(w2t - w2k) * gi ** 2 + 2 * w2k * gi ** 2 * eg
    bias1_t, bias1_k = 1.0 - beta1 ** step, 1.0 - b1f ** step
    bias2_t, bias2_k = 1.0 - beta2 ** step, 1.0 - b2f ** step
    vi = ref["exp_avg_sq"][0]
    with np.errstate(divide="ignore", invalid="ignore"):
        rel_v = np.where(vi > 0, dv / vi, 0.0)
    upd = np.abs(ref["update"][0])
    sqrt_part = 0.5 * (rel_v + abs(bias2_t - bias2_k) / bias2_k)
    return (float(lr) / bias1_k * dm / ref["denom"][0]
            + upd * (abs(bias1_t - bias1_k) / bias1_k + sqrt_part)) * 1.01
