"""The float64 restatement of the one-launch single-agent rollout's forward and selection
(tests/sa_forward_reference.py) on a machine without a GPU: it equals the torch modules in
float64, its float32 bound holds for an emulation of the kernel's arithmetic and rejects
seeded faults, its search_index equals the C oracle's sampler, and the kernel's support query
agrees with an independent restatement of its shape envelope."""
import ctypes
import itertools

import numpy as np
import pytest
import torch

import sa_forward_reference as R
from mlp_reference import bf16_rne

# (F, hidden widths, A): non-square layers, three hidden layers, odd widths, the widest policy
SHAPES = [(4, [32, 32], 2), (6, [64, 48, 16], 3), (2, [7], 3), (3, [9, 33, 63], 1),
          (6, [64, 64, 64], 3), (2, [1, 8], 1), (4, [], 2)]
FAULTS = ["drop_last", "neighbour_bias", "relu_head", "transpose", "bf16"]
MAX_WEIGHTS = 11 * 1024          # floats of shared memory the kernel gives the policy
MAX_WIDTH = 64


class _Env:
    """What FullyConnected / FullyConnectedActor read from an EnvWrapper (no device needed)."""

    class _DM:
        def get_shape(self, name=None):
            return (8, 4, 1, 3)

    def __init__(self, F, A, continuous):
        from warp_drive_b200.utils import spaces

        act = (spaces.Box(-2.0, 2.0, shape=(A,), dtype=np.float32) if continuous
               else spaces.Discrete(A))

        class _E:
            observation_space = {0: spaces.Box(-1.0, 1.0, shape=(F,), dtype=np.float32)}
            action_space = {0: act}

        self.env = _E()
        self.n_agents = 1
        self.cuda_data_manager = self._DM()


def _obs(rows, F, seed=0):
    return np.random.default_rng(seed + 100).standard_normal((rows, F)).astype(np.float32)


def emulate(obs, layers, continuous, scale=1.0, bias=0.0, fault=None, fault_layer=0):
    """The kernel's float32 arithmetic in numpy: every neuron one chain bias, + w[0] x[0],
    + w[1] x[1], ... (each step the exact float64 product plus the add, rounded to float32),
    fmaxf ReLU; softmax as max subtraction, exp, sequential sum and division; or
    fl(fl(scale * tanh(z)) + bias).  exp and tanh are rounded from float64 (correctly rounded
    here, within the 2 ulp the bound allows the device).  `fault` seeds one mistake."""
    f32, f64 = np.float32, np.float64
    x = np.asarray(obs, f32)
    for l, (w, b) in enumerate(layers):
        w, b = np.asarray(w, f32), np.asarray(b, f32)
        if fault == "bf16":
            w = bf16_rne(w)
        if l == fault_layer and fault == "transpose":
            assert w.shape[0] == w.shape[1]
            w = np.ascontiguousarray(w.T)
        if l == fault_layer and fault == "neighbour_bias":
            b = np.roll(b, -1)
        n = w.shape[1] - (1 if fault == "drop_last" and l == fault_layer else 0)
        acc = np.broadcast_to(b, (x.shape[0], w.shape[0])).astype(f32)
        for i in range(n):
            acc = (acc.astype(f64) + x[:, i:i + 1].astype(f64) * w[None, :, i].astype(f64)
                   ).astype(f32)
        if l < len(layers) - 1 or fault == "relu_head":
            acc = np.maximum(acc, f32(0))
        x = acc
    if continuous:
        t = np.tanh(x.astype(f64)).astype(f32)
        return f32(scale) * t + f32(bias)
    e = np.exp((x - x.max(-1, keepdims=True)).astype(f64)).astype(f32)
    s = np.zeros(x.shape[0], f32)
    for i in range(x.shape[1]):
        s = s + e[:, i]
    return e / s[:, None]


def _torch_module(F, hidden, A, layers, continuous, scale, bias):
    from warp_drive_b200.training.models.fully_connected import ModelFactory

    kind = "fully_connected_actor" if continuous else "fully_connected"
    cfg = {"type": kind, "fc_dims": list(hidden), "output_w": scale, "output_b": bias,
           "model_ckpt_filepath": ""}
    m = ModelFactory.create(kind)(env=_Env(F, A, continuous), model_config=cfg, policy="shared",
                                  policy_tag_to_agent_id_map={"shared": [0]}).double()
    linears = [m.fc[str(i)][0] for i in range(len(m.fc))]
    linears.append(m.policy_head if continuous else m.policy_head[0])
    with torch.no_grad():
        for lin, (w, b) in zip(linears, layers):
            lin.weight.copy_(torch.from_numpy(w.astype(np.float64)))
            lin.bias.copy_(torch.from_numpy(b.astype(np.float64)))
    return m


@pytest.mark.parametrize("continuous", [False, True])
@pytest.mark.parametrize("F,hidden,A", [s for s in SHAPES if s[1]])
def test_reference_equals_the_torch_modules_in_float64(F, hidden, A, continuous):
    A = 1 if continuous else max(A, 2)
    layers = R.make_policy([F] + hidden + [A], scale=3.0, seed=F + len(hidden))
    m = _torch_module(F, hidden, A, layers, continuous, 2.0, 0.25)
    obs = _obs(257, F)
    with torch.no_grad():
        got = m(torch.from_numpy(obs.astype(np.float64)))
    got = (got[0] if continuous else got[0][0]).numpy()
    want = R.forward(obs, layers, continuous, 2.0, 0.25)["out"]
    assert got.shape == want.shape
    assert np.abs(got - want).max() <= 1e-12


def _cases():
    for F, hidden, A in SHAPES:
        for continuous in (False, True):
            yield F, hidden, (1 if continuous else max(A, 2)), continuous


@pytest.mark.parametrize("F,hidden,A,continuous", list(_cases()))
@pytest.mark.parametrize("scale", [1.0, 10.0, 100.0])
def test_float32_emulation_lies_within_the_bound(F, hidden, A, continuous, scale):
    layers = R.make_policy([F] + hidden + [A], scale=scale, seed=7)
    obs = _obs(512, F, seed=1)
    ref = R.forward(obs, layers, continuous, 2.0, 0.25)
    got = emulate(obs, layers, continuous, 2.0, 0.25).astype(np.float64)
    err = np.abs(got - ref["out"])
    assert (err <= ref["bound"]).all(), float((err / ref["bound"]).max())
    assert (got[ref["zero"]] == 0).all()


@pytest.mark.parametrize("continuous", [False, True])
@pytest.mark.parametrize("fault", FAULTS)
def test_seeded_faults_exceed_the_bound(fault, continuous):
    A = 1 if continuous else 3
    # (F, hidden widths, faulty layer); only the first has a square layer (32 -> 32)
    for F, hidden, layer in ((6, [32, 32], 1), (4, [9, 33, 7], 2), (3, [16], 0)):
        if fault == "transpose" and hidden != [32, 32]:
            continue
        layers = R.make_policy([F] + hidden + [A], scale=1.0, seed=3)
        obs = _obs(256, F, seed=2)
        ref = R.forward(obs, layers, continuous, 2.0, 0.25)
        bad = emulate(obs, layers, continuous, 2.0, 0.25, fault=fault, fault_layer=layer)
        err = np.abs(bad.astype(np.float64) - ref["out"])
        assert (err > ref["bound"]).any(), (fault, F, hidden)


def _supported_restated(n_hidden, dims):
    if not 0 <= n_hidden <= 3:
        return 0
    d = dims[:n_hidden + 2]
    if any(w < 1 or w > MAX_WIDTH for w in d):
        return 0
    total = sum(d[l] * d[l + 1] + d[l + 1] for l in range(n_hidden + 1))
    return int(total <= MAX_WEIGHTS)


def test_support_query_agrees_with_the_restated_envelope(wdb_lib):
    widths = [0, 1, 2, 7, 8, 9, 31, 32, 33, 63, 64, 65]
    arr = (ctypes.c_int * 6)()
    q = wdb_lib.wdb_single_agent_rollout_supported
    counts = {0: 0, 1: 0}
    for n_hidden in range(-1, 5):
        n = min(max(n_hidden + 2, 1), 6)
        for dims in itertools.product(widths, repeat=n):
            for i, v in enumerate(dims):
                arr[i] = v
            want = _supported_restated(n_hidden, list(dims))
            assert q(n_hidden, arr) == want, (n_hidden, dims)
            counts[want] += 1
    assert counts[0] > 0 and counts[1] > 0
    # the weight cap: F -> 64 -> 64 -> h3 -> A around 11 264 floats
    F, h3, A = np.meshgrid(np.arange(1, 65), np.arange(1, 65), np.arange(1, 65), indexing="ij")
    total = (F * 64 + 64) + (64 * 64 + 64) + (64 * h3 + h3) + (h3 * A + A)
    for delta in (-1, 0, 1):
        hits = np.argwhere(total == MAX_WEIGHTS + delta)
        assert len(hits), delta
        for f, h, a in hits[:64] + 1:
            for i, v in enumerate((f, 64, 64, h, a)):
                arr[i] = int(v)
            assert q(3, arr) == (1 if delta <= 0 else 0), (f, h, a)
    # the widest policy the discrete kinds need fits; a NULL dims array is refused
    for i, v in enumerate((6, 64, 64, 64, 3)):
        arr[i] = v
    assert q(3, arr) == 1
    assert q(1, None) == 0


def _rows():
    """(p, u) rows that reach every branch of the search."""
    rows = []
    flat = [0.25, 0.0, 0.0, 0.5, 0.25]                       # flat CDF steps
    for u in (0.25, 0.2, 0.3, 0.75, 0.7500001, 1.0, 1e-9, 0.0):
        rows.append((flat, u))
    lead0 = [0.0, 0.0, 1.0]                                   # zeros first: u below 1e-8
    for u in (1e-9, 1e-7, 0.5, 1.0):
        rows.append((lead0, u))
    short = np.array([0.2, 0.2, 0.2], np.float32)            # float32 total below 1
    for p in (np.full(3, 1 / 3, np.float32), short, np.full(10, 0.1, np.float32)):
        tot = np.cumsum(p, dtype=np.float32)[-1]
        for u in (1.0, np.nextafter(tot, np.float32(2)), tot, 0.9):
            rows.append((p, u))
    g = np.random.default_rng(11)
    for _ in range(300):
        A = int(g.integers(1, 13))
        p = g.random(A).astype(np.float32)
        p[g.random(A) < 0.3] = 0
        if p.sum() == 0:
            p[-1] = 1
        p = (p / p.sum()).astype(np.float32)
        cdf = np.cumsum(p, dtype=np.float32)
        for u in list(cdf) + [p[0] * 0.5, g.random(), 1.0, cdf[0] + 5e-9]:
            rows.append((p, u))
    return rows


def test_search_index_equals_the_c_oracle(oracle_lib):
    rows = _rows()
    for A in sorted({len(p) for p, _ in rows}):
        sel = [(np.asarray(p, np.float32), np.float32(u)) for p, u in rows if len(p) == A]
        P = np.stack([p for p, _ in sel])
        u = np.array([u for _, u in sel], np.float32)
        for argmax in (0, 1):
            out = np.zeros(len(sel), np.int32)
            oracle_lib.wd_oracle_sample_actions(P, out, 1, None, u, len(sel), A, argmax)
            want = R.argmax_first(P) if argmax else R.search_index(P, u)
            assert (out == want).all(), (A, argmax, P[out != want], u[out != want])


def test_search_index_branches():
    """Hand-checked selections: flat steps return the probe the search meets first, u = 1.0 and u
    above a float32 total below 1 clamp to the last index, u below p[0] is index 0."""
    flat = np.array([0.25, 0.0, 0.0, 0.5, 0.25], np.float32)
    assert R.search_index(flat, np.float32(0.25)) == 2        # first probe mid = 2 hits 0.25
    assert R.search_index(flat, np.float32(0.3)) == 3
    assert R.search_index(flat, np.float32(0.2)) == 0
    assert R.search_index(flat, np.float32(1.0)) == 4
    short = np.array([0.2, 0.2, 0.2], np.float32)
    assert R.search_index(short, np.float32(0.9)) == 2
    assert R.search_index(np.array([0.0, 0.0, 1.0], np.float32), np.float32(1e-9)) == 1
    assert R.argmax_first(np.array([0.1, 0.45, 0.45], np.float32)) == 1
