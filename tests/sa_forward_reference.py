"""Float64 restatement of the one-launch single-agent rollout's policy forward and action
selection (wdb_single_agent_rollout, csrc/wdb_sa_rollout.cu), written from the operations'
definitions rather than from the kernel, with an a-priori bound on how far the kernel's float32
arithmetic may land from it.

Forward: n_hidden (0..3) Linear + ReLU layers (nn.Linear weights [out, in]), then the head:
softmax(z) for the discrete kinds, action_scale * tanh(z) + action_bias for the continuous ones.

Bound.  U = 2**-24 is float32's unit roundoff, gamma_n = n U / (1 - n U), TINY = 2**-149 the
smallest subnormal.  The library is built without -ftz and without fast math, so subnormals are
kept: a rounded product or quotient r errs by at most U |r| + TINY / 2, a rounded sum by at most
U |r| (a sum that lands in the subnormal range is exact).

1. Pre-activations.  Every neuron is one fmaf chain s_0 = b, s_k = fl(s_{k-1} + w_k x^_k),
   k = 1 .. n (n = fan-in; the lanes split neurons, not the sum, so the order is fixed).  Its n
   roundings give, by the recursive-summation argument,
       |s^ - (b + sum w x^)| <= gamma_n (|b| + sum |w| |x^|) + n TINY.
   The kernel's inputs x^ differ from the float64 activations x by at most e_x (0 for the
   observation: both read the same float32 row), so |x^| <= |x| + e_x and
       e_z = gamma_n (|b| + sum |w| (|x| + e_x)) + sum |w| e_x + n TINY.
   ReLU is 1-Lipschitz, so the activation's error is e_z again.
2. Softmax head (logits z_i with errors e_i, E = max_i e_i, m = max z, d_i = z_i - m <= 0):
   - m^ = max z^ is exact (fmaxf) and |m^ - m| <= E;
   - d^_i = fl(z^_i - m^), one rounding:
         |d^_i - d_i| <= D_i = e_i + E + U (|d_i| + e_i + E);
   - x_i = expf(d^_i), at most 2 ulp from exp(d^_i) (CUDA Programming Guide, single-precision
     mathematical functions); 2 ulp <= 4U |y| for a normal y and <= 2 TINY below:
         |x_i - exp(d_i)| <= c_i = exp(d_i) ((1 + 4U) exp(D_i) - 1) + 2 TINY;
   - S^ = the sequential float32 sum of the A positive x_i, A - 1 roundings after the exact
     first add (S = sum exp(d_i) >= 1):
         |S^ - S| <= s = sum c_i + gamma_{A-1} sum (exp(d_i) + c_i),
     and S^ >= 1 as well: the largest logit gives d^ = 0 exactly and expf(0) = 1, and a
     rounded sum of non-negative terms never falls below one of them;
   - p^_i = fl(x_i / S^), IEEE division:
         |p^_i - p_i| <= (c_i + p_i s + U (exp(d_i) + c_i)) / max(S - s, 1) + TINY / 2.
3. Tanh head: tanhf is at most 2 ulp from tanh and tanh is 1-Lipschitz, so
       |t^ - tanh z| <= e_t = e_z + 4U (|tanh z| + e_z) + 2 TINY,
   and mean^ = fl(fl(action_scale t^) + action_bias) carries two more roundings:
       |mean^ - mean| <= |scale| e_t + gamma_2 (|scale| (|tanh z| + e_t) + |bias|) + TINY.

Selection (search_index of the reference's sampler, core/random.cu): the float32 CDF in
sequential order, a binary search that returns a probe within 1e-8 of u at once, otherwise the
first index whose CDF value is >= u, clamped to the last index.  Argmax: the first maximum wins.
"""
import numpy as np

U = 2.0 ** -24
TINY = 2.0 ** -149
EPS_SEARCH = np.float32(1e-8)


def gamma(n):
    n = np.asarray(n, np.float64)
    return n * U / (1 - n * U)


def make_policy(dims, scale=1.0, seed=0):
    """[(W [out, in], b [out])] in float32 for layer widths `dims` = [F, H1, ..., A]: He-scaled
    uniform hidden layers (activations stay O(1) through the ReLUs) and a head whose logits are
    about +-`scale` (1 .. 100 spans soft to saturated heads)."""
    g = np.random.default_rng(seed)
    layers = []
    for l in range(len(dims) - 1):
        fan_in, out = dims[l], dims[l + 1]
        a = np.sqrt(6.0 / fan_in)
        if l == len(dims) - 2:
            a *= scale
        w = g.uniform(-a, a, (out, fan_in)).astype(np.float32)
        b = g.uniform(-0.5, 0.5, out).astype(np.float32)
        layers.append((w, b))
    return layers


def _trunk(obs, layers):
    """float64 logits and their error bound (section 1 of the module docstring)."""
    x = np.asarray(obs, np.float64)
    ex = np.zeros_like(x)
    for l, (w, b) in enumerate(layers):
        w = np.asarray(w, np.float64)
        b = np.asarray(b, np.float64)
        n = w.shape[1]
        aw = np.abs(w)
        z = x @ w.T + b
        ez = gamma(n) * (np.abs(b) + (np.abs(x) + ex) @ aw.T) + ex @ aw.T + n * TINY
        if l < len(layers) - 1:
            x, ex = np.maximum(z, 0.0), ez
        else:
            return z, ez


def _softmax(z, ez):
    A = z.shape[-1]
    E = ez.max(-1, keepdims=True)
    d = z - z.max(-1, keepdims=True)
    D = ez + E + U * (np.abs(d) + ez + E)
    e = np.exp(d)
    c = e * (np.expm1(D) + 4 * U * np.exp(D)) + 2 * TINY
    S = e.sum(-1, keepdims=True)
    s = c.sum(-1, keepdims=True) + gamma(A - 1) * (e + c).sum(-1, keepdims=True)
    p = e / S
    bound = (c + p * s + U * (e + c)) / np.maximum(S - s, 1.0) + TINY / 2
    # exp(d^_i) < TINY / 2 for every d^_i the bound allows: expf rounds it to 0, so p^_i = 0
    zero = np.exp(d + D) * (1 + 4 * U) < TINY / 2
    return p, bound, zero


def _tanh_head(z, ez, scale, bias):
    t = np.tanh(z)
    et = ez + 4 * U * (np.abs(t) + ez) + 2 * TINY
    mean = scale * t + bias
    bound = abs(scale) * et + gamma(2) * (abs(scale) * (np.abs(t) + et) + abs(bias)) + TINY
    return mean, bound


def forward(obs, layers, continuous=False, action_scale=1.0, action_bias=0.0):
    """dict(out=probs [rows, A] or mean [rows, 1], bound=its float32 error bound,
    z / ez = logits and their bound, zero = where the kernel's probability must be 0)."""
    z, ez = _trunk(obs, layers)
    if continuous:
        out, bound = _tanh_head(z, ez, float(action_scale), float(action_bias))
        zero = np.zeros(out.shape, bool)
    else:
        out, bound, zero = _softmax(z, ez)
    return {"out": out, "bound": bound, "z": z, "ez": ez, "zero": zero}


def ou_reference(mean, mean_bound, normals, ou0, damping, stddev, scale):
    """float64 actions mean_t + scale ((1 - damping) ou_{t-1} + stddev n_t) and their bound,
    the OU state carried over [T, E] timesteps from ou0.  The kernel rounds 1 - damping, the
    product with ou, stddev * n and their sum (or fuses the last two into one fma): at most three
    roundings on the ou term and two on the noise term, then the product with scale and the add
    of the mean (or one fma)."""
    d, sd, sc = float(np.float32(damping)), float(np.float32(stddev)), float(np.float32(scale))
    a = 1.0 - d
    ou = np.asarray(ou0, np.float64).copy()
    eou = np.zeros_like(ou)
    acts, bounds = [], []
    for t in range(len(normals)):
        nz = sd * np.asarray(normals[t], np.float64)
        s = a * ou + nz
        es = a * eou + gamma(3) * (a * (np.abs(ou) + eou) + np.abs(nz)) + 2 * TINY
        m, em = mean[t], mean_bound[t]
        acts.append(m + sc * s)
        bounds.append(em + sc * es + gamma(2) * (np.abs(m) + em + sc * (np.abs(s) + es)) + TINY)
        ou, eou = s, es
    return np.stack(acts), np.stack(bounds)


def search_index(p, u):
    """The sampler's index for float32 rows p [..., A] and uniforms u [...]: sequential float32
    CDF, binary search with the |cdf - u| < 1e-8 shortcut, clamp to A - 1."""
    p = np.asarray(p, np.float32)
    u = np.asarray(u, np.float32)
    A = p.shape[-1]
    cdf = np.cumsum(p, axis=-1, dtype=np.float32)      # add.accumulate: strictly in order
    left = np.zeros(u.shape, np.int64)
    right = np.full(u.shape, A - 1, np.int64)
    found = np.full(u.shape, -1, np.int64)
    while True:
        active = (left <= right) & (found < 0)
        if not active.any():
            break
        mid = left + (right - left) // 2
        v = np.take_along_axis(cdf, np.clip(mid, 0, A - 1)[..., None], -1)[..., 0]
        hit = active & (np.abs(v - u) < EPS_SEARCH)
        found = np.where(hit, mid, found)
        up = active & ~hit & (v < u)
        down = active & ~hit & ~(v < u)
        left = np.where(up, mid + 1, left)
        right = np.where(down, mid - 1, right)
    return np.where(found >= 0, found, np.minimum(left, A - 1))


def argmax_first(p):
    """Index of the first maximum of each row (a later equal value does not replace it)."""
    return np.argmax(np.asarray(p), axis=-1)


def categorical_float64(p, bound, u):
    """(index, decided) of the float64 categorical choice: the first i with cdf_i >= u, and
    whether u lies far enough from every float64 CDF value that the kernel's float32 CDF (each
    p^ within `bound`, plus the sum's own roundings) and the 1e-8 shortcut cannot choose
    otherwise."""
    A = p.shape[-1]
    cdf = np.cumsum(p, axis=-1)
    cb = np.cumsum(bound, axis=-1) + gamma(np.arange(A)) * np.cumsum(p + bound, axis=-1)
    u = np.asarray(u, np.float64)[..., None]
    idx = np.minimum((cdf < u).sum(-1), A - 1)
    decided = (np.abs(cdf - u) > cb + 2 * float(EPS_SEARCH)).all(-1)
    return idx, decided


def argmax_float64(p, bound):
    """(index, decided): the float64 argmax, and whether its lead over every other entry
    exceeds both bounds, so that the kernel's float32 probabilities have the same first max."""
    top = np.argmax(p, axis=-1)
    pt = np.take_along_axis(p, top[..., None], -1)
    bt = np.take_along_axis(bound, top[..., None], -1)
    lead = (pt - p > bt + bound)
    np.put_along_axis(lead, top[..., None], True, -1)
    return top, lead.all(-1)
