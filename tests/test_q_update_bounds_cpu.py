"""tests/q_update_bounds.py on the CPU: its values are those of the float64 references of the
DQN-family passes, a float32 torch evaluation of each pass (algorithms/dqn.py's losses, another
summation order than the kernels') lies within its bars, and its per-element bars reject small
defects that a norm-wise 2e-4 check accepts.  The case builders here feed
tests/test_gpu_q_update_exact.py too."""
import copy

import numpy as np
import pytest
import torch

import c51_reference as cref
import dqn_update_reference as dref
import iqn_reference as iref
import per_reference as pref
import q_update_bounds as qb
import qr_dqn_reference as qref
from test_ddpg_update_reference_cpu import layers

GAMMA = 0.97


def _f32(x):
    return float(np.float32(x))


def _models(kind, F, A, dims, N=1, iqn=None, seed=0):
    """(online, target) float32 models; the target perturbed away from the online network."""
    if kind == "dqn":
        q, t = dref.make_q_models(F, A, dims, seed=seed)
    elif kind == "qr" and N == 1:
        # the model takes N >= 2; the pass takes N = 1, DQN's network with one quantile
        q, t = dref.make_q_models(F, A, dims, seed=seed)
        q.num_quantiles = t.num_quantiles = 1
    elif kind == "qr":
        q, t = qref.make_qr_models(F, A, N, dims, seed=seed)
    elif kind == "c51":
        q, t = cref.make_c51_models(F, A, dims, N=N, v_min=-3.0, v_max=4.0, seed=seed)
    else:
        n_cos, n_tau, n_tau_prime, K = iqn
        q, t = iref.make_iqn_models(F, A, dims, n_cos=n_cos, N=n_tau, NP=n_tau_prime, K=K,
                                    seed=seed)
    with torch.no_grad():
        for p in t.parameters():
            p.add_(0.3 * torch.randn_like(p))
        if kind == "iqn":
            for net in (q, t):                   # most embedding units active
                net.tau_embedding.bias.add_(0.3)
    return q.float(), t.float()


def _ring(C, E, Np, F, A, seed):
    obs, actions, rewards, done = dref.make_q_ring(C, E, Np, F, A, seed)
    return [obs.astype(np.float32), actions, rewards.astype(np.float32), done]


def _f64_layers(model):
    return [(w.astype(np.float64), b.astype(np.float64)) for w, b in layers(model)]


class Case:
    """One pass on one shape: the float32 models, the ring, B windows (and IQN's taus) whose
    every premise holds, kappa / delta, the weights, and the bar reference of each launch."""

    def __init__(self, kind, B, n_step, C, E, Np, F, A, dims, N=1, iqn=None, gamma=GAMMA,
                 double_q=True, seed=None, models=None):
        """models: float32 (online, target) to use instead of fresh ones of this shape."""
        seed = B if seed is None else seed
        self.kind, self.B, self.n_step, self.C, self.E, self.Np = kind, B, n_step, C, E, Np
        self.N, self.iqn, self.double_q, self.gamma = N, iqn, double_q, _f32(gamma)
        self.models = _models(kind, F, A, dims, N, iqn, seed) if models is None else models
        self.ring = _ring(C, E, Np, F, A, seed)
        g = np.random.default_rng(seed)
        n = 2 * B + 64
        w = np.stack([g.integers(0, C, n), g.integers(0, E * Np, n)], axis=1).astype(np.int32)
        w[0] = (C - 1, E * Np - 1)                       # wraps the physical end of the ring
        self.taus = None
        if kind == "iqn":
            self.taus = g.uniform(0.0, 1.0, (n, iqn[1] + iqn[2])).astype(np.float32)
        self.kappa = 1.0
        probe = self.reference(w, self.taus, kappa=1e9 if kind == "dqn" else 1.0)
        if kind == "dqn":
            diff = np.abs(probe["q_values"][0] - probe["returns"][0])
            self.kappa = _f32(np.median(diff) + 1e-3)
        elif kind in ("qr", "iqn"):
            self.kappa = _f32(np.median(np.abs(self._u(w))) + 1e-3)
        ok = self.reference(w, self.taus)["ok"]
        keep = np.flatnonzero(ok)
        if len(keep) < B:
            pytest.fail(f"only {len(keep)} of {n} drawn windows satisfy every premise; {B} needed")
        keep = keep[:B]
        self.windows = w[keep].copy()
        if self.taus is not None:
            self.taus = self.taus[keep].copy()
        if B > 2:                                        # a duplicate window
            self.windows[2] = self.windows[1]
            if self.taus is not None:
                self.taus[2] = self.taus[1]
        self.weights = g.uniform(0.1, 1.0, B).astype(np.float32)

    def _u(self, w):
        if self.kind == "qr":
            return qref.qr_dqn_sampled(self.models, self.ring, w, self.n_step, self.gamma, 1.0,
                                       self.double_q, self.N)["u"]
        return iref.iqn_sampled(self.models, self.ring, w, self.n_step, self.gamma, 1.0,
                                self.double_q, self.taus)["u"]

    def rows(self, w):
        return dref.gather(self.ring, w, self.n_step, self.Np)

    def support(self):
        q = self.models[0]
        return q.support.detach().cpu().float().numpy(), np.float32(q.delta_z)

    def reference(self, w=None, taus=None, weights=None, kappa=None):
        w = self.windows if w is None else w
        taus = self.taus if taus is None else taus
        kappa = self.kappa if kappa is None else kappa
        rows = self.rows(w)
        q, t = self.models
        if self.kind in ("dqn", "qr"):
            return qb.qr_pass(_f64_layers(q), _f64_layers(t), rows, self.gamma, kappa,
                              self.double_q, self.N, weights, dqn=self.kind == "dqn")
        if self.kind == "c51":
            z, dz = self.support()
            return qb.c51_pass(_f64_layers(q), _f64_layers(t), rows, self.gamma, self.double_q,
                               z, dz, weights)
        pq, pt = iref.parts(q), iref.parts(t)
        return qb.iqn_pass(pq[0], pq[1], pq[2], pt[0], pt[1], pt[2], rows, self.gamma, kappa,
                           self.double_q, taus, self.iqn[1], self.iqn[3], weights)

    def existing(self, weights=None):
        """The existing float64 reference's dict on the same float32 inputs."""
        m, w = [copy.deepcopy(x).double() for x in self.models], self.windows
        if self.kind == "dqn":
            if weights is None:
                return dref.dqn_sampled(m, self.ring, w, self.n_step, self.gamma, self.kappa,
                                        self.double_q)
            return pref.dqn_weighted(m, self.ring, w, weights, self.n_step, self.gamma,
                                     self.kappa, self.double_q)
        if self.kind == "qr":
            return qref.qr_dqn_sampled(m, self.ring, w, self.n_step, self.gamma, self.kappa,
                                       self.double_q, self.N, weights)
        if self.kind == "c51":
            z, dz = self.support()
            return cref.c51_sampled(m, self.ring, w, self.n_step, self.gamma, self.double_q,
                                    z.astype(np.float64), float(dz), weights)
        return iref.iqn_sampled(m, self.ring, w, self.n_step, self.gamma, self.kappa,
                                self.double_q, self.taus, weights)


def within(got, ref, what):
    """Every element of got within its bar of the value (exactly the value where the bar is 0);
    returns the largest |err| / bar."""
    v, b = ref
    got = np.asarray(got, dtype=np.float64).reshape(np.shape(v))
    err = np.abs(got - v)
    bad = ~(err <= b)
    if bad.any():
        i = np.unravel_index(int(np.argmax(np.where(bad, err - b, -np.inf))), np.shape(v))
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} elements outside their bar;"
                             f" worst at {i}: got {got[i]!r}, value {v[i]!r}, bar {b[i]!r}")
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(b > 0, err / b, 0.0)
    return float(r.max()) if r.size else 0.0


def _values(kind, ref, old):
    keys = {"dqn": ("q", "returns", "sum_huber"), "qr": ("qbar", "rbar", "sum_loss"),
            "c51": ("qbar", "rbar", "sum_loss"), "iqn": ("qbar", "rbar", "sum_loss")}[kind]
    pairs = [(a[0], b) for a, b in zip(ref["grads"], old["grads"])]
    pairs += [(ref["q_values"][0], old[keys[0]]), (ref["returns"][0], old[keys[1]]),
              (ref["sums"][0][0], old[keys[2]]), (ref["sums"][1][0], old["sum_q"])]
    for got, want in pairs:
        got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
        scale = max(float(np.abs(want).max()) if want.size else 0.0, 1e-300)
        assert float(np.abs(got - want).max() if want.size else 0.0) <= 1e-12 * scale


# (kind, B, n_step, C, E, Np, F, A, dims, N, iqn (n_cos, N, N', K), gamma)
VALUE_CASES = [
    ("dqn", 1, 3, 9, 4, 1, 4, 2, [64, 64], 1, None, GAMMA),
    ("dqn", 300, 1, 5, 3, 3, 6, 3, [16], 1, None, 0.0),
    ("dqn", 40, 2, 12, 4, 1, 63, 1, [5, 7, 9], 1, None, 1.0),
    ("dqn", 17, 3, 12, 4, 1, 4, 3, [], 1, None, GAMMA),
    ("qr", 17, 3, 12, 4, 1, 4, 2, [1], 1, None, GAMMA),
    ("qr", 60, 3, 12, 4, 1, 4, 1, [64, 64], 64, None, GAMMA),
    ("c51", 17, 3, 12, 4, 1, 4, 2, [64, 64], 51, None, GAMMA),
    ("c51", 40, 2, 12, 4, 3, 4, 3, [5, 7, 9], 2, None, 1.0),
    ("c51", 40, 3, 12, 4, 1, 4, 1, [], 64, None, GAMMA),
    ("iqn", 17, 3, 12, 4, 1, 4, 2, [64, 64], 1, (64, 8, 8, 256), GAMMA),
    ("iqn", 9, 2, 12, 4, 1, 4, 3, [5, 7, 9], 1, (1, 1, 64, 1), 0.0),
]


def _case_id(c):
    return f"{c[0]}_B{c[1]}_A{c[7]}_L{len(c[8])}_N{c[9]}" + (f"_iqn{'-'.join(map(str, c[10]))}"
                                                             if c[10] else "")


def make_case(c, double_q):
    kind, B, n_step, C, E, Np, F, A, dims, N, iqn, gamma = c
    return Case(kind, B, n_step, C, E, Np, F, A, dims, N, iqn, gamma, double_q)


@pytest.mark.parametrize("weighted", [False, True], ids=["uniform", "weighted"])
@pytest.mark.parametrize("double_q", [True, False], ids=["double_q", "max_target"])
@pytest.mark.parametrize("c", VALUE_CASES, ids=[_case_id(c) for c in VALUE_CASES])
def test_values_match_the_existing_references(c, double_q, weighted):
    case = make_case(c, double_q)
    wt = case.weights if weighted else None
    _values(case.kind, case.reference(weights=wt), case.existing(wt))


@pytest.mark.parametrize("A,N,S", [(1, 1, 4), (3, 1, 0), (2, 51, 32), (3, 13, 8), (4, 64, 0)])
def test_fold_and_unfold_values_match_the_dueling_reference(A, N, S):
    import dueling_reference as dueling
    from test_dueling_cpu import make_dueling

    head = make_dueling(4, A, N, [7], S, seed=A + N + S).float().policy_head
    p = dueling.stream_params(head)
    for got, want in zip(qb.fold(p, A, N, S), dueling.fold(p, A, N, S)):
        for g, w in zip(got, want):
            assert np.abs(g[0] - w).max() <= 1e-12 * np.abs(w).max() and (g[1] >= 0).all()
    g = np.random.default_rng(A * N + S)
    grads = [(g.standard_normal(w.shape).astype(np.float32), g.standard_normal(b.shape)
              .astype(np.float32)) for w, b in dueling.fold(p, A, N, S)]
    got, want = qb.unfold(grads, A, N, S), dueling.unfold(
        [(w.astype(np.float64), b.astype(np.float64)) for w, b in grads], A, N, S)
    assert got.keys() == want.keys()
    for k in want:
        assert np.abs(got[k][0] - want[k]).max() <= 1e-12 * max(np.abs(want[k]).max(), 1e-30)


# ------------------------------------------------------------------------ soundness
def _torch_grads(case, weights):
    """Float32 torch autograd through algorithms/dqn.py's loss on the case's windows."""
    from warp_drive_b200.training.algorithms import dqn as algos

    q, t = case.models
    obs, actions, rewards, done, boot = (torch.from_numpy(np.ascontiguousarray(x))
                                         for x in case.rows(case.windows))
    obs, boot, rewards = obs.float(), boot.float(), rewards.float()
    kw = {}
    if case.kind == "dqn":
        algo = algos.DQN(case.gamma, n_step=case.n_step, double_q=case.double_q,
                         huber_delta=case.kappa)
    elif case.kind == "qr":
        algo = algos.QuantileDQN(case.gamma, n_step=case.n_step, double_q=case.double_q,
                                 huber_delta=case.kappa)
    elif case.kind == "iqn":
        algo = algos.ImplicitQuantileDQN(case.gamma, n_step=case.n_step, double_q=case.double_q,
                                         huber_delta=case.kappa)
        kw["taus"] = torch.from_numpy(case.taus)
    else:
        algo = algos.CategoricalDQN(case.gamma, n_step=case.n_step, double_q=case.double_q)
    w = None if weights is None else torch.from_numpy(weights)
    loss, qv, ret = algo.loss(q, t, obs, actions.reshape(-1, 1), rewards, done,
                              boot, w, **kw)
    grads = torch.autograd.grad(loss, list(q.parameters()))
    return [g.double().numpy() for g in grads], qv.detach().double().numpy(), \
        ret.detach().double().numpy()


# CartPole-like shapes whose support spacing is a float32 (torch divides by the Python float)
SOUND_CASES = [
    ("dqn", 97, 3, 12, 4, 1, 4, 2, [64, 64], 1, None, GAMMA),
    ("qr", 97, 3, 12, 4, 1, 4, 2, [16, 16], 8, None, GAMMA),
    ("c51", 97, 3, 12, 4, 1, 4, 2, [16, 16], 2, None, GAMMA),
    ("iqn", 33, 3, 12, 4, 1, 4, 2, [16, 16], 1, (8, 4, 5, 6), GAMMA),
]


@pytest.mark.parametrize("weighted", [False, True], ids=["uniform", "weighted"])
@pytest.mark.parametrize("c", SOUND_CASES, ids=[_case_id(c) for c in SOUND_CASES])
def test_a_float32_torch_update_lies_within_the_bars(c, weighted):
    case = make_case(c, True)
    if case.kind == "c51":                       # dz = 7: a float32, as torch divides by it
        assert float(np.float32(case.models[0].delta_z)) == case.models[0].delta_z
    wt = case.weights if weighted else None
    ref = case.reference(weights=wt)
    grads, qv, ret = _torch_grads(case, wt)
    names = [n for n, _ in case.models[0].named_parameters()]
    for name, got, want in zip(names, grads, ref["grads"]):
        within(got, want, name)
    if case.kind == "dqn":                       # the others' torch means are float32 sums
        within(qv, ref["q_values"], "q_values")
        within(ret, ref["returns"], "returns")


# ------------------------------------------------------------------------ sensitivity
def _norm_ok(got, value):
    return float(np.linalg.norm(got - value) / max(np.linalg.norm(value), 1e-30)) <= 2e-4


def _bars_ok(got, ref):
    v, b = ref
    return bool((np.abs(got - v) <= b).all())


def test_per_element_bars_reject_defects_the_norm_wise_check_accepts():
    # C51 at the run config's shape: B = 333, CartPole, [64, 64], N = 51, double_q
    c51 = Case("c51", 333, 3, 40, 6, 1, 4, 2, [64, 64], 51, None, GAMMA, True)
    ref = c51.reference()
    head_w = ref["grads"][-2]
    v = head_w[0]
    small = np.abs(v) < 2e-4 * np.linalg.norm(v)
    assert small.sum() > 100
    # zero the small elements, smallest first, as far as the norm-wise check still accepts
    order = np.argsort(np.abs(v), axis=None)
    got = v.copy()
    zeroed = 0
    for i in order:
        trial = got.copy()
        trial.flat[i] = 0.0
        if not _norm_ok(trial, v) or not small.flat[i]:
            break
        got, zeroed = trial, zeroed + 1
    assert zeroed > 100 and _norm_ok(got, v) and not _bars_ok(got, head_w)
    # scale a whole tensor by (1 + 1e-4): DQN's second-layer weights at the same shape (C51's
    # bars, carried through its softmax differences, are too wide relative to this slip)
    dqn = Case("dqn", 333, 3, 40, 6, 1, 4, 2, [64, 64], 1, None, GAMMA, True)
    g = dqn.reference()["grads"][2]
    got = g[0] * (1 + 1e-4)
    assert _norm_ok(got, g[0]) and not _bars_ok(got, g)
    # a gross defect both checks reject: drop atom 7 of every action from the head
    got = v.copy()
    got[7::51] = 0.0
    assert not _norm_ok(got, v) and not _bars_ok(got, head_w)

    # IQN at the same shape, n_cos = 64, N = N' = K = 32
    iqn = Case("iqn", 333, 3, 40, 6, 1, 4, 2, [64, 64], 1, (64, 32, 32, 32), GAMMA, True)
    ref = iqn.reference()
    emb_w = ref["grads"][-2]
    v, b = emb_w
    cand = np.flatnonzero(((np.abs(v) < 2e-4 * np.linalg.norm(v)) & (np.abs(v) > b)).ravel())
    assert cand.size
    got = v.copy()
    got.flat[cand[0]] = -got.flat[cand[0]]           # one small element's sign flipped
    assert _norm_ok(got, v) and not _bars_ok(got, emb_w)
    # a dead unit's exact-zero gradient made a small non-zero value
    trunk_w = ref["grads"][2]
    zeros = np.flatnonzero((trunk_w[1] == 0).ravel() & (trunk_w[0] == 0).ravel())
    assert zeros.size
    got = trunk_w[0].copy()
    got.flat[zeros[0]] = 1e-12 * np.abs(trunk_w[0]).max()
    assert _norm_ok(got, trunk_w[0]) and not _bars_ok(got, trunk_w)
