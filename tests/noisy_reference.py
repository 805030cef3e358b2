"""Float64 NumPy restatement of noisy networks' noise and maps (include/wdb200.h wdb_noisy_*;
models/fully_connected_q.py NoisyLinear): the noise element on the documented Philox counter
(oracle.philox4x32_10, as per_reference.philox_words), the effective layer and the gradient map."""
import numpy as np

TAG = 0x4E000000
UPDATE, ACTING = 0, 1


def counter(domain, count, row, layer, e):
    """The Philox counter words of noise element e."""
    return [count & 0xFFFFFFFF, TAG | (domain << 16) | ((count >> 32) & 0xFFFF), row,
            (layer << 16) | (e >> 1)]


def noise(seed, domain, count, row, layer, n):
    """(f(eps), bar) of elements 0 .. n - 1: f in float64 from the float32 uniforms and the
    float32 angle the kernel forms, and the per-element bound of the float32 evaluation -- logf
    (1 ulp), sqrtf (rounded), cosf (2 ulp), the product and f's sqrtf, relative to |f|."""
    import oracle

    key = [seed & 0xFFFFFFFF, seed >> 32]
    f = np.zeros(n)
    for e in range(n):
        w = oracle.philox4x32_10(counter(domain, count, row, layer, e), key)
        a, b = (int(w[0]), int(w[1])) if e % 2 == 0 else (int(w[2]), int(w[3]))
        u1 = np.float32(np.float32(a) * np.float32(2.0 ** -32) + np.float32(2.0 ** -33))
        u2 = np.float32(np.float32(b) * np.float32(2.0 ** -32) + np.float32(2.0 ** -33))
        angle = np.float32(np.float32(6.2831853071795864) * u2)
        x = np.sqrt(-2.0 * np.log(np.float64(u1))) * np.cos(np.float64(angle))
        f[e] = np.sign(x) * np.sqrt(abs(x))
    return f, 1e-6 * np.abs(f)


def layer_noise(seed, domain, count, row, layer, n_in, n_out):
    """(f(eps_in) [in], f(eps_out) [out]) of one noisy layer."""
    f, _ = noise(seed, domain, count, row, layer, n_in + n_out)
    return f[:n_in], f[n_in:]


def materialize(mu_w, sigma_w, mu_b, sigma_b, fi, fo):
    """The effective (W, b)."""
    return mu_w + sigma_w * np.outer(fo, fi), mu_b + sigma_b * fo


def grads(dw, db, fi, fo):
    """(d mu_W, d sigma_W, d mu_b, d sigma_b) from the effective layer's gradients."""
    return dw, dw * np.outer(fo, fi), db, db * fo


def factored(x, mu_w, sigma_w, mu_b, sigma_b, fi, fo):
    """The per-row forward y = mu_W x + mu_b + fo * (sigma_W (fi * x) + sigma_b); fi [R, in],
    fo [R, out] (or vectors)."""
    return x @ mu_w.T + mu_b + fo * ((fi * x) @ sigma_w.T + sigma_b)
