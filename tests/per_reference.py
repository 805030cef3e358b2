"""Float64 NumPy restatement of prioritized replay (include/wdb200.h, wdb_per_*; csrc/wdb_per.cu)
and of the importance-weighted DQN update (wdb_dqn_update_prioritized) on top of
tests/dqn_update_reference.py: the sum tree in the kernel's child order, the admit ranges, the
stratified descent fed by oracle.philox4x32_10 words, the weights and the priorities."""
import numpy as np

import dqn_update_reference as dqn_ref

FAN = 32


def build_tree(leaves):
    """The float64 node levels over float32 leaves, parents of the leaves first, root last:
    each node is its 32 zero-padded children summed pairwise, v[i] += v[i + h] for h = 16 .. 1
    (bit for bit what the kernels compute)."""
    level = np.asarray(leaves, dtype=np.float32).astype(np.float64)
    levels = []
    while True:
        n = -(-len(level) // FAN)
        v = np.zeros(n * FAN)
        v[:len(level)] = level
        v = v.reshape(n, FAN)
        h = FAN // 2
        while h >= 1:
            v[:, :h] = v[:, :h] + v[:, h:2 * h]
            h //= 2
        level = v[:, 0].copy()
        levels.append(level)
        if n == 1:
            return levels


def flat_nodes(levels):
    """The levels as the device array wdb_per_store.nodes holds them."""
    return np.concatenate(levels)


def n_levels(n_leaves):
    return len(build_tree(np.zeros(n_leaves, dtype=np.float32)))


def valid_starts(C, oldest, filled, n_step):
    """Boolean [C]: physical slots whose window is valid (logical start k in [0, filled - n_step
    - 1])."""
    k = (np.arange(C) - oldest) % C
    return k <= filled - n_step - 1


def admit(leaves, p_max, alpha, C, n_rows, n_step, before, after):
    """wdb_per_admit on a copy of leaves [C * n_rows] (float32): the starts that just became
    valid get p_max^alpha, the newest n_step slots 0."""
    out = np.array(leaves, dtype=np.float32).reshape(C, n_rows)
    (c0, _), (c1, f1) = before, after
    T = (c1 - c0) % C
    oldest = c1 if f1 == C else 0
    ok = valid_starts(C, oldest, f1, n_step)
    enter = np.float32(np.power(np.float32(p_max), np.float32(alpha)))
    for j in range(T + n_step):
        s = (c1 - n_step - T + j) % C
        out[s] = enter if (j < T and ok[s]) else np.float32(0)
    return out.reshape(-1)


def uniform53(words):
    """[B, 4] uint32 Philox words -> the 53-bit uniform in [0, 1) of the sampler."""
    w = np.asarray(words, dtype=np.uint64)
    return ((w[:, 0] >> 5).astype(np.float64) * 67108864.0
            + (w[:, 1] >> 6).astype(np.float64)) * (1.0 / 9007199254740992.0)


def philox_words(seed, counter, B):
    """[B, 4] words of Philox4x32-10 with key seed at counter (counter, g)."""
    import oracle

    key = [seed & 0xFFFFFFFF, seed >> 32]
    return np.array([oracle.philox4x32_10(
        [counter & 0xFFFFFFFF, counter >> 32, g & 0xFFFFFFFF, g >> 32], key)
        for g in range(B)], dtype=np.uint64)


def segment_points(S, u01):
    """Row g's point lo + U (hi - lo) of the stratum [g S / B, (g + 1) S / B)."""
    B = len(u01)
    g = np.arange(B, dtype=np.float64)
    lo = (g * S) / B
    hi = ((g + 1) * S) / B
    return lo + u01 * (hi - lo), lo, hi


def descend(leaves, levels, u):
    """The leaf each point u [B] reaches (the kernel's scan: running prefix, first positive
    child whose prefix end exceeds u, else the last positive child)."""
    leaves64 = np.asarray(leaves, dtype=np.float32).astype(np.float64)
    below = [leaves64] + levels[:-1]          # the children of level l's nodes
    B = len(u)
    u = np.array(u, dtype=np.float64)
    node = np.zeros(B, dtype=np.int64)
    for l in reversed(range(len(levels))):
        child = below[l]
        sel = np.full(B, -1, dtype=np.int64)
        base = np.zeros(B)
        last = node * FAN
        last_base = np.zeros(B)
        prefix = np.zeros(B)
        for k in range(FAN):
            c = node * FAN + k
            inside = c < len(child)
            v = np.where(inside, child[np.minimum(c, len(child) - 1)], 0.0)
            nxt = prefix + v
            pos = inside & (v > 0)
            take = pos & (sel < 0) & (u < nxt)
            sel = np.where(take, c, sel)
            base = np.where(take, prefix, base)
            last = np.where(pos, c, last)
            last_base = np.where(pos, prefix, last_base)
            prefix = nxt
        none = sel < 0
        sel = np.where(none, last, sel)
        base = np.where(none, last_base, base)
        u = u - base
        node = sel
    return node


def sample(leaves, n_rows, B, seed, counter):
    """(windows [B, 2] int32, priorities [B] float32, the points u [B]) of
    wdb_per_sample_windows."""
    levels = build_tree(leaves)
    u, _, _ = segment_points(levels[-1][0], uniform53(philox_words(seed, counter, B)))
    leaf = descend(leaves, levels, u)
    windows = np.stack([leaf // n_rows, leaf % n_rows], axis=1).astype(np.int32)
    return windows, np.asarray(leaves, dtype=np.float32)[leaf], u


def weights(priorities, beta):
    """(p_g / min p)^-beta in float64."""
    p = np.asarray(priorities, dtype=np.float64)
    return (p / p.min()) ** (-float(beta))


def brute_force_leaf(leaves, u):
    """The leaf whose float64 cumulative interval [prefix, prefix + p) holds u, over the
    positive leaves in index order (the last positive leaf for u past the total)."""
    p = np.asarray(leaves, dtype=np.float32).astype(np.float64)
    ends = np.cumsum(p)
    pos = np.flatnonzero(p > 0)
    idx = np.searchsorted(ends[pos], u, side="right")
    return pos[np.minimum(idx, len(pos) - 1)]


def priorities(q, returns, alpha, eps):
    """(|Q - R| + eps)^alpha in float64."""
    return (np.abs(np.asarray(q, np.float64) - np.asarray(returns, np.float64)) + eps) ** alpha


def set_priorities(leaves, p_max, windows, q, returns, alpha, eps, C, n_rows, n_step, oldest,
                   filled):
    """wdb_per_set_priorities on copies (float32 leaves, p_max): duplicates keep the largest."""
    out = np.array(leaves, dtype=np.float32)
    ok = valid_starts(C, oldest, filled, n_step)
    p = (np.abs(np.asarray(q, np.float32) - np.asarray(returns, np.float32))
         + np.float32(eps)).astype(np.float32)
    v = np.power(p, np.float32(alpha)).astype(np.float32)
    new = {}
    for g, (s, n) in enumerate(windows):
        if ok[s]:
            leaf = int(s) * n_rows + int(n)
            new[leaf] = max(new.get(leaf, np.float32(0)), v[g])
            p_max = max(p_max, p[g])
    for leaf, val in new.items():
        out[leaf] = val
    return out, np.float32(p_max)


def dqn_weighted(models, ring, windows, w, n_step, gamma, delta, double_q):
    """dqn_update_reference.dqn_sampled with importance-sampling weights w [B]: the loss
    (1/B) sum w_g huber_g and its gradients ({"grads", "sum_huber" (weighted), "q", "returns",
    "sum_q", "diff"})."""
    from test_ddpg_update_reference_cpu import layers

    base = dqn_ref.dqn_sampled(models, ring, windows, n_step, gamma, delta, double_q)
    Lq = layers(models[0])
    Np = ring[0].shape[2]
    obs, actions, _, _, _ = dqn_ref.gather(ring, windows, n_step, Np)
    B = obs.shape[0]
    w = np.asarray(w, dtype=np.float64)
    diff = base["diff"]
    ad = np.abs(diff)
    huber = np.where(ad < delta, 0.5 * diff * diff, delta * (ad - 0.5 * delta))
    qs, inputs = dqn_ref.forward(Lq, obs)
    d = np.zeros_like(qs)
    d[np.arange(B), actions] = w * np.clip(diff, -delta, delta) / B
    grads = [None] * len(Lq)
    for i in reversed(range(len(Lq))):
        wi, _ = Lq[i]
        grads[i] = (d.T @ inputs[i], d.sum(axis=0))
        if i > 0:
            d = (d @ wi) * (inputs[i] > 0)
    return {"grads": [g for pair in grads for g in pair], "sum_huber": float((w * huber).sum()),
            "q": base["q"], "returns": base["returns"], "sum_q": base["sum_q"], "diff": diff}
