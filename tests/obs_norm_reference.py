"""NumPy restatement of the observation statistics and normalization (csrc/wdb_obs_norm.cu).

Moments are float64 (n, mean, M2) per feature: Welford row by row for a small batch, and for a
large one each fixed row range's moments (two-pass) merged in range order by Chan et al.'s
formula, as the device merges its per-CTA records.  The normalization restates the kernel's
float32 operations in its order: a rounded subtract, a rounded multiply, then the clamp.
"""
import numpy as np


def welford(x):
    """(n, mean [F], M2 [F]) of x [rows, F], float64 Welford over the rows in order."""
    x = np.asarray(x, dtype=np.float64).reshape(-1, np.shape(x)[-1])
    n, mean, m2 = 0, np.zeros(x.shape[1]), np.zeros(x.shape[1])
    for row in x:
        n += 1
        d = row - mean
        mean = mean + d / n
        m2 = m2 + d * (row - mean)
    return float(n), mean, m2


def moments(x):
    """(n, mean, M2) of x [rows, F] in float64, two-pass."""
    x = np.asarray(x, dtype=np.float64).reshape(-1, np.shape(x)[-1])
    if x.shape[0] == 0:
        return 0.0, np.zeros(x.shape[1]), np.zeros(x.shape[1])
    mean = x.mean(axis=0)
    return float(x.shape[0]), mean, ((x - mean) ** 2).sum(axis=0)


def chan(a, b):
    """Merge two (n, mean, M2) triples; an empty side leaves the other as it is."""
    na, ma, m2a = a
    nb, mb, m2b = b
    if nb == 0:
        return a
    if na == 0:
        return b
    n = na + nb
    d = mb - ma
    return n, ma + d * (nb / n), m2a + m2b + d * d * (na * nb / n)


def batch_moments(x, n_ranges=None):
    """(n, mean, M2) of x [rows, F]: fixed row ranges (the device's split by default) merged in
    order."""
    x = np.asarray(x, dtype=np.float32).reshape(-1, np.shape(x)[-1])
    rows = x.shape[0]
    p = n_ranges or device_records(rows)
    out = (0.0, np.zeros(x.shape[1]), np.zeros(x.shape[1]))
    for r in range(p):
        out = chan(out, moments(x[r * rows // p:(r + 1) * rows // p]))
    return out


def device_records(rows):
    """Per-CTA records of the device's partial pass: one per 1024 rows, at most 512."""
    return int(min(512, max(1, -(-rows // 1024))))


def shift_scale(n, mean, m2):
    """float32 (shift, scale) of the statistics: (0, 1) with no samples, else (mean,
    1 / sqrt(M2 / n + 1e-8)) rounded from float64."""
    mean = np.asarray(mean, dtype=np.float64)
    if n == 0:
        return np.zeros(mean.shape, np.float32), np.ones(mean.shape, np.float32)
    var = np.asarray(m2, dtype=np.float64) / n
    return mean.astype(np.float32), (1.0 / np.sqrt(var + 1e-8)).astype(np.float32)


def normalize_f32(x, shift, scale, clip):
    """clamp((x - shift) * scale, -clip, clip) in float32, the kernel's operations in order."""
    x = np.asarray(x, dtype=np.float32)
    y = np.subtract(x, np.asarray(shift, np.float32), dtype=np.float32)
    y = np.multiply(y, np.asarray(scale, np.float32), dtype=np.float32)
    c = np.float32(clip)
    return np.minimum(np.maximum(y, -c), c)
