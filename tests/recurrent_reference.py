"""NumPy float64 restatement of FullyConnectedGRU (training/models/fully_connected_gru.py):

* `forward_sequence` with the reset rule h_in(t) = h_out(t - 1) * (1 - [done(t - 1) > 0]);
* its BPTT gradients for the loss sum_k <cp_k, probs_k> + <cv, values> (no gradient into h0);
* `step_with_bounds`: one rollout step and, per output, an a-priori bound on how far
  wdb_gru_policy_forward's float32 result (csrc/wdb_recurrent.cu) may lie from it.

Parameters are a dict of float64 arrays keyed by the model's state_dict names."""
import numpy as np

U = 2.0 ** -24            # float32 unit roundoff


def params_of(model):
    return {k: v.detach().cpu().double().numpy() for k, v in model.state_dict().items()}


def _n_layers(P):
    return sum(1 for k in P if k.startswith("fc.") and k.endswith(".0.weight"))


def _n_heads(P):
    return sum(1 for k in P if k.startswith("policy_head.") and k.endswith(".weight"))


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def _softmax(x):
    e = np.exp(x - x.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def _cell(P, x, h):
    """nn.GRUCell: (h', cache)."""
    H = h.shape[-1]
    gi = x @ P["gru.weight_ih"].T + P["gru.bias_ih"]
    gh = h @ P["gru.weight_hh"].T + P["gru.bias_hh"]
    r = _sigmoid(gi[:, :H] + gh[:, :H])
    z = _sigmoid(gi[:, H:2 * H] + gh[:, H:2 * H])
    n = np.tanh(gi[:, 2 * H:] + r * gh[:, 2 * H:])
    return (1 - z) * n + z * h, (x, h, gh, r, z, n)


def _trunk(P, obs):
    acts = [obs]
    for i in range(_n_layers(P)):
        acts.append(np.maximum(acts[-1] @ P[f"fc.{i}.0.weight"].T + P[f"fc.{i}.0.bias"], 0.0))
    return acts


def forward_sequence(P, obs, h0, done):
    """obs [T, E, Np, F], h0 [E, Np, H], done [T, E] -> (probs per head [T, E, Np, A_k],
    values [T, E, Np], cache)."""
    T, E, Np, F = obs.shape
    H = h0.shape[-1]
    acts = _trunk(P, obs.reshape(T, E * Np, F))
    x = acts[-1]
    h = h0.reshape(E * Np, H)
    hs, caches, keeps = [], [], []
    for t in range(T):
        keep = np.ones(E * Np)
        if t > 0:
            keep = np.repeat((done[t - 1] <= 0).astype(np.float64), Np)
            h = h * keep[:, None]
        keeps.append(keep)
        h, c = _cell(P, x[t], h)
        hs.append(h)
        caches.append(c)
    hs = np.stack(hs)                                       # [T, R, H]
    probs = [_softmax(hs @ P[f"policy_head.{k}.weight"].T + P[f"policy_head.{k}.bias"])
             for k in range(_n_heads(P))]
    values = (hs @ P["vf_head.weight"].T + P["vf_head.bias"])[..., 0]
    shape = (T, E, Np)
    return ([p.reshape(shape + (-1,)) for p in probs], values.reshape(shape),
            (acts, hs, caches, keeps))


def gradients(P, obs, h0, done, cp, cv):
    """d/dtheta of sum_k <cp[k], probs_k> + <cv, values> (cp[k] [T, E, Np, A_k], cv [T, E, Np])
    by backpropagation through time; h0 is a constant.  {state_dict name: gradient}."""
    T, E, Np, F = obs.shape
    R = E * Np
    probs, _, (acts, hs, caches, keeps) = forward_sequence(P, obs, h0, done)
    G = {k: np.zeros_like(v) for k, v in P.items()}
    dh_all = np.zeros_like(hs)
    for k, p in enumerate(probs):
        p = p.reshape(T, R, -1)
        c = cp[k].reshape(T, R, -1)
        dl = p * (c - (c * p).sum(-1, keepdims=True))          # softmax backward
        G[f"policy_head.{k}.weight"] += np.einsum("tra,trh->ah", dl, hs)
        G[f"policy_head.{k}.bias"] += dl.sum((0, 1))
        dh_all += dl @ P[f"policy_head.{k}.weight"]
    dv = cv.reshape(T, R, 1)
    G["vf_head.weight"] += np.einsum("tro,trh->oh", dv, hs)
    G["vf_head.bias"] += dv.sum((0, 1))
    dh_all += dv @ P["vf_head.weight"]
    H = hs.shape[-1]
    Wih, Whh = P["gru.weight_ih"], P["gru.weight_hh"]
    dx = np.zeros((T, R, Wih.shape[1]))
    carry = np.zeros((R, H))
    for t in range(T - 1, -1, -1):
        x, h, gh, r, z, n = caches[t]
        dh = dh_all[t] + carry
        dn = dh * (1 - z)
        dz = dh * (h - n)
        dh_prev = dh * z
        dan = dn * (1 - n * n)                                  # pre-tanh
        dgi_n = dan
        dgh_n = dan * r
        dr = dan * gh[:, 2 * H:]
        dar = dr * r * (1 - r)
        daz = dz * z * (1 - z)
        dgi = np.concatenate([dar, daz, dgi_n], -1)
        dgh = np.concatenate([dar, daz, dgh_n], -1)
        G["gru.weight_ih"] += dgi.T @ x
        G["gru.bias_ih"] += dgi.sum(0)
        G["gru.weight_hh"] += dgh.T @ h
        G["gru.bias_hh"] += dgh.sum(0)
        dx[t] = dgi @ Wih
        dh_prev = dh_prev + dgh @ Whh
        carry = dh_prev * keeps[t][:, None]                     # the reset before step t
    g = dx.reshape(T * R, -1)
    for i in range(_n_layers(P) - 1, -1, -1):
        a_out = acts[i + 1].reshape(T * R, -1)
        a_in = acts[i].reshape(T * R, -1)
        g = g * (a_out > 0)
        G[f"fc.{i}.0.weight"] += g.T @ a_in
        G[f"fc.{i}.0.bias"] += g.sum(0)
        g = g @ P[f"fc.{i}.0.weight"]
    return G


def _gamma(n):
    return n * U / (1 - n * U)


def _dense_bound(W, b, x, ex):
    """y = W x + b on rows x [R, K] carrying errors ex: (y, bound) of the kernel's k-ascending
    fmaf sum of x-hat (|x-hat - x| <= ex) plus the bias."""
    K = W.shape[1]
    aW = np.abs(W)
    y = x @ W.T + b
    mag = (np.abs(x) + ex) @ aW.T + np.abs(b)
    return y, ex @ aW.T + _gamma(K + 1) * mag


def step_with_bounds(P, obs, h):
    """One wdb_gru_policy_forward step in float64: obs [R, F], h [R, H] ->
    (probs per head [R, A_k], h' [R, H], their bounds).  The bounds propagate each float32
    operation's rounding (u = 2^-24; expf and tanhf within 2 ulp) and the inputs' errors to first
    order through the Lipschitz constants of ReLU (1), the sigmoid (1/4), tanh (1) and the
    softmax (2 max|dl| relative); a factor 2 covers the second-order terms."""
    x, ex = obs, np.zeros_like(obs)
    for i in range(_n_layers(P)):
        y, ey = _dense_bound(P[f"fc.{i}.0.weight"], P[f"fc.{i}.0.bias"], x, ex)
        x, ex = np.maximum(y, 0.0), ey
    H = h.shape[-1]
    gi, egi = _dense_bound(P["gru.weight_ih"], P["gru.bias_ih"], x, ex)
    gh, egh = _dense_bound(P["gru.weight_hh"], P["gru.bias_hh"], h, np.zeros_like(h))
    sl = {g: slice(j * H, (j + 1) * H) for j, g in enumerate("rzn")}

    def gate(g):
        a = gi[:, sl[g]] + gh[:, sl[g]]
        ea = egi[:, sl[g]] + egh[:, sl[g]] + U * np.abs(a)
        s = _sigmoid(a)
        return s, 0.25 * ea + 6 * U * s
    r, er = gate("r")
    z, ez = gate("z")
    ghn, eghn = gh[:, sl["n"]], egh[:, sl["n"]]
    prod = r * ghn
    eprod = er * np.abs(ghn) + np.abs(r) * eghn + er * eghn + U * np.abs(prod)
    a = gi[:, sl["n"]] + prod
    ea = egi[:, sl["n"]] + eprod + U * np.abs(a)
    n = np.tanh(a)
    en = ea + 4 * U * np.abs(n)
    hn = (1 - z) * n + z * h
    ehn = ez * (np.abs(n) + np.abs(h)) + (1 - z + ez) * en + 4 * U * (
        np.abs((1 - z) * n) + np.abs(z * h))
    ehn = 2 * ehn
    probs, eprobs = [], []
    for k in range(_n_heads(P)):
        W, b = P[f"policy_head.{k}.weight"], P[f"policy_head.{k}.bias"]
        logit, el = _dense_bound(W, b, hn, ehn)
        p = _softmax(logit)
        A = logit.shape[-1]
        spread = np.abs(logit - logit.max(-1, keepdims=True)).max(-1, keepdims=True)
        rel = 2 * el.max(-1, keepdims=True) + 2 * U * spread + 8 * U + _gamma(A)
        probs.append(p)
        eprobs.append(2 * p * rel)
    return probs, hn, eprobs, ehn
