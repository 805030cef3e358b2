"""NumPy float64 restatement of FullyConnectedGaussianGRU (training/models/fully_connected_gru.py),
built on tests/recurrent_reference.py's trunk, cell and bounds:

* `gaussian_forward_sequence`: the sequence forward with the reset rule, the mean head raw;
* `gaussian_gradients`: its BPTT gradients for a loss given by its gradients with respect to the
  mean, the values and log_std (no gradient into h0);
* `gaussian_step_with_bounds`: one rollout step of wdb_gru_policy_forward's mean head kind and,
  per output, an a-priori bound on how far its float32 result may lie from it.

Parameters are a dict of float64 arrays keyed by the model's state_dict names."""
import numpy as np

from recurrent_reference import _dense_bound, _n_layers, forward_sequence, step_with_bounds


def _categorical_stand_in(P):
    """P with the mean head swapped for a one-action softmax head, so that forward_sequence runs
    the shared trunk and cell of a Gaussian model's parameters."""
    Q = {k: v for k, v in P.items() if not k.startswith("policy_head.") and k != "log_std"}
    H = P["policy_head.weight"].shape[1]
    Q["policy_head.0.weight"], Q["policy_head.0.bias"] = np.zeros((1, H)), np.zeros(1)
    return Q


def gaussian_forward_sequence(P, obs, h0, done):
    """FullyConnectedGaussianGRU.forward_sequence: obs [T, E, Np, F], h0 [E, Np, H], done [T, E]
    -> (mean [T, E, Np, A], values [T, E, Np], cache)."""
    _, values, cache = forward_sequence(_categorical_stand_in(P), obs, h0, done)
    hs = cache[1]
    mean = hs @ P["policy_head.weight"].T + P["policy_head.bias"]
    return mean.reshape(values.shape + (-1,)), values, cache


def gaussian_gradients(P, obs, h0, done, g_mean, g_values, g_log_std):
    """d/dtheta of a loss with dloss/dmean = g_mean [T, E, Np, A], dloss/dvalues = g_values
    [T, E, Np] and dloss/dlog_std = g_log_std [A], by backpropagation through time; h0 is a
    constant.  {state_dict name: gradient}."""
    T, E, Np, F = obs.shape
    R = E * Np
    _, _, (acts, hs, caches, keeps) = gaussian_forward_sequence(P, obs, h0, done)
    G = {k: np.zeros_like(v) for k, v in P.items()}
    G["log_std"] = np.asarray(g_log_std, np.float64).copy()
    dm = g_mean.reshape(T, R, -1)
    G["policy_head.weight"] += np.einsum("tra,trh->ah", dm, hs)
    G["policy_head.bias"] += dm.sum((0, 1))
    dv = g_values.reshape(T, R, 1)
    G["vf_head.weight"] += np.einsum("tro,trh->oh", dv, hs)
    G["vf_head.bias"] += dv.sum((0, 1))
    dh_all = dm @ P["policy_head.weight"] + dv @ P["vf_head.weight"]
    H = hs.shape[-1]
    Wih, Whh = P["gru.weight_ih"], P["gru.weight_hh"]
    dx = np.zeros((T, R, Wih.shape[1]))
    carry = np.zeros((R, H))
    for t in range(T - 1, -1, -1):
        x, h, gh, r, z, n = caches[t]
        dh = dh_all[t] + carry
        dan = dh * (1 - z) * (1 - n * n)                        # pre-tanh
        daz = dh * (h - n) * z * (1 - z)
        dar = dan * gh[:, 2 * H:] * r * (1 - r)
        dgi = np.concatenate([dar, daz, dan], -1)
        dgh = np.concatenate([dar, daz, dan * r], -1)
        G["gru.weight_ih"] += dgi.T @ x
        G["gru.bias_ih"] += dgi.sum(0)
        G["gru.weight_hh"] += dgh.T @ h
        G["gru.bias_hh"] += dgh.sum(0)
        dx[t] = dgi @ Wih
        carry = (dh * z + dgh @ Whh) * keeps[t][:, None]         # the reset before step t
    g = dx.reshape(T * R, -1)
    for i in range(_n_layers(P) - 1, -1, -1):
        g = g * (acts[i + 1].reshape(T * R, -1) > 0)
        G[f"fc.{i}.0.weight"] += g.T @ acts[i].reshape(T * R, -1)
        G[f"fc.{i}.0.bias"] += g.sum(0)
        g = g @ P[f"fc.{i}.0.weight"]
    return G


def gaussian_step_with_bounds(P, obs, h):
    """One wdb_gru_policy_forward step of the mean head kind in float64: obs [R, F], h [R, H] ->
    (mean [R, A], h' [R, H], their bounds).  h' and its bound are step_with_bounds'; the mean is
    the head's k-ascending fmaf sum plus bias on h', bounded by _dense_bound from h's bound."""
    _, hn, _, ehn = step_with_bounds(_categorical_stand_in(P), obs, h)
    mean, emean = _dense_bound(P["policy_head.weight"], P["policy_head.bias"], hn, ehn)
    return mean, hn, emean, ehn
