"""`wdb_single_agent_rollout`'s in-kernel policy forward and action selection against the float64
restatement (tests/sa_forward_reference.py), driven through the C ABI so that every shape the
kernel accepts is reachable (0..3 hidden layers of width 1..64, which the torch modules cannot
all express): every recorded probability (the mean, for the continuous kinds) within the
a-priori float32 bound of the float64 forward of the recorded observation; the sampled index
equal to the restated search_index on the kernel's own probabilities, bit for bit; two launches
from the same state bit-identical; nothing written outside the arrays the kernel owns, in
particular past row E - 1 of a partly filled CTA; malformed policies refused without a launch."""
import ctypes

import numpy as np
import pytest
import torch

import sa_forward_reference as R
import test_gpu_ddpg_rollout as ddpg_rollout
import test_gpu_single_agent_rollout as sa_rollout

pytestmark = pytest.mark.gpu

GUARD = 64
SENTINEL = {torch.float32: 12345.0, torch.int32: 0x5EED5EED, torch.int64: 0x5EED5EED5EED}
OU = {"damping": 0.3, "stddev": 0.5, "scale": 0.8}
ACTION_SCALE, ACTION_BIAS = 2.0, 0.25
# kind (WDB_SA_*) -> (env name in the rollout test modules, observation width, action count)
KINDS = {0: ("cartpole", 4, 2), 1: ("mountain_car", 2, 3), 2: ("acrobot", 6, 3),
         3: ("continuous_mountain_car", 2, 1), 4: ("pendulum", 3, 1)}
EPISODE = 8
T = 2 * EPISODE + 4                  # every replica resets at least twice
WIDTHS = [1, 7, 8, 9, 33, 63, 64]
# the arrays of the env the kernel writes: struct field -> data manager name
ENV_ARRAYS = {"state": "state", "observations": "observations", "done": "_done_",
              "env_timestep": "_timestep_", "rewards": "rewards",
              "sampled_actions": "sampled_actions"}


def _hidden(kind, n_hidden):
    """n_hidden widths drawn from WIDTHS, each layer with a different fan-in and fan-out."""
    g = np.random.default_rng(10 * kind + n_hidden)
    F, A = KINDS[kind][1], KINDS[kind][2]
    out, prev = [], F
    for i in range(n_hidden):
        last = i == n_hidden - 1
        w = int(g.choice([x for x in WIDTHS if x != prev and not (last and x == A)]))
        out.append(w)
        prev = w
    return out


CASES = []   # (kind, hidden widths, E, reset pool size, logit scale, family)
for _k in KINDS:
    for _n in range(4):
        CASES.append((_k, _hidden(_k, _n), [1, 7, 9, 61][(_k + _n) % 4], 8 * (_n % 2),
                      [1.0, 10.0, 100.0][(_k + _n) % 3], f"hidden{_n}"))
    CASES.append((_k, [64, 64, 64], 61, 8, 30.0, "widest"))
CASES += [(0, [32, 32], 10_000, 8, 1.0, "config3"),
          (0, [64, 64, 64], 10_000, 0, 100.0, "widest"),
          (4, [64, 64, 64], 10_000, 8, 10.0, "widest")]

_ENGINES = {}


def _engine(kind, E, pool):
    key = (kind, E, pool)
    if key not in _ENGINES:
        name = KINDS[kind][0]
        mod = ddpg_rollout if kind >= 3 else sa_rollout
        w, eng, s, _ = mod._build(name, E, 1, pool, fused=True, episode_length=EPISODE)
        assert eng.sa is not None
        _ENGINES[key] = (w, eng, s)
    return _ENGINES[key]


def _guarded(shape, dtype, guards):
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * GUARD,), SENTINEL[dtype], dtype=dtype, device="cuda")
    guards.append(buf)
    return buf[GUARD:GUARD + n].view(shape)


class Run:
    """A wdb_sa_rollout that owns every array the kernel writes (sentinel-guarded copies of the
    env's current rows, fresh batch slots and sums), the policy `layers`, a reset table that
    restores into those copies and copies of the RNG states, so that every launch starts from
    the same state and leaves the env untouched."""

    def __init__(self, kind, E, pool, layers, n_steps=T):
        from warp_drive_b200 import lib as wlib
        from warp_drive_b200.utils.constants import Constants as C

        self.wlib = wlib
        self.kind, self.E, self.n_steps = kind, E, n_steps
        self.continuous = kind >= 3
        w, eng, s = _engine(kind, E, pool)
        self.dm = dm = w.cuda_data_manager
        self.base = eng.sa.r
        self.init = {f: dm.data_on_device_via_torch(n).clone() for f, n in ENV_ARRAYS.items()}
        if self.continuous:
            self.init["ou_state"] = dm.data_on_device_via_torch(f"{C.ACTIONS}_ou_state").clone()
        self.env_ptr = {f: wlib.ptr(dm.data_on_device_via_torch(n))
                        for f, n in ENV_ARRAYS.items()}
        self.rng0 = s.rng_state.clone()
        table, self.n_reset, pool_rng = eng.sa._reset_table()
        self.table_bytes = table.cpu().numpy().tobytes()
        self.pool0 = None if pool_rng is None else pool_rng.clone()
        self.layers = [(torch.from_numpy(wt).cuda(), torch.from_numpy(b).cuda())
                       for wt, b in layers]
        self.dims = [layers[0][0].shape[1]] + [wt.shape[0] for wt, _ in layers]

    def struct(self):
        """A fresh struct with fresh guarded arrays; returns (struct, arrays, guard buffers)."""
        wlib = self.wlib
        r = wlib.SaRollout.from_buffer_copy(self.base)
        E, Tn = self.E, self.n_steps
        F, A = self.dims[0], self.dims[-1]
        arrays, guards = {}, []

        def own(field, src):
            view = _guarded(tuple(src.shape), src.dtype, guards)
            view.copy_(src)
            arrays[field] = view
            setattr(r, field, wlib.ptr(view))

        for field, src in self.init.items():
            own(field, src)
        act = torch.float32 if self.continuous else torch.int32
        for field, shape, dtype in (("obs_batch", (Tn, E, F), torch.float32),
                                    ("actions_batch", (Tn, E), act),
                                    ("rewards_batch", (Tn, E), torch.float32),
                                    ("done_batch", (Tn, E), torch.int32),
                                    ("probs_batch", (Tn, E) if self.continuous else (Tn, E, A),
                                     torch.float32),
                                    ("reward_running_sum", (E,), torch.float32),
                                    ("step_running_sum", (E,), torch.int32),
                                    ("episodic_reward_sum", (1,), torch.float32),
                                    ("episodic_step_sum", (1,), torch.int64),
                                    ("num_completed", (1,), torch.int64)):
            own(field, torch.zeros(shape, dtype=dtype, device="cuda"))
        r.n_steps = Tn
        r.n_hidden = len(self.layers) - 1
        for i in range(5):
            r.dims[i] = self.dims[i] if i < len(self.dims) else 0
        for i in range(4):
            r.w[i], r.b[i] = (wlib.ptr(self.layers[i][0]), wlib.ptr(self.layers[i][1])) \
                if i < len(self.layers) else (None, None)
        keep = [self.rng0.clone()]
        r.rng_state = wlib.ptr(keep[0])
        if self.pool0 is not None:
            keep.append(self.pool0.clone())
            r.pool_rng = wlib.ptr(keep[-1])
        # the reset table, its targets moved to the copies
        n = self.n_reset
        if n:
            desc = (wlib.ResetDesc * n).from_buffer_copy(self.table_bytes[:n * ctypes.sizeof(
                wlib.ResetDesc)])
            back = {p: f for f, p in self.env_ptr.items()}
            for i in range(n):
                assert desc[i].dst in back, "a reset target the test does not own"
                desc[i].dst = wlib.ptr(arrays[back[desc[i].dst]])
            table = torch.frombuffer(bytearray(bytes(desc)), dtype=torch.uint8).cuda()
            keep.append(table)
            r.reset_table, r.n_reset_arrays = wlib.ptr(table), n
        r.reset_done_envs = 1
        r.uniforms = r.normals = None
        r.use_argmax = 0
        if self.continuous:
            r.action_scale, r.action_bias = ACTION_SCALE, ACTION_BIAS
            r.ou_damping, r.ou_stddev, r.ou_scale = OU["damping"], OU["stddev"], OU["scale"]
        self._keep = keep
        return r, arrays, guards

    def launch(self, uniforms=None, normals=None, use_argmax=False):
        wlib = self.wlib
        r, arrays, guards = self.struct()
        r.uniforms = wlib.ptr(uniforms)
        r.normals = wlib.ptr(normals)
        r.use_argmax = int(use_argmax)
        wlib.check(wlib.load().wdb_single_agent_rollout(wlib.stream_ptr(), ctypes.byref(r)),
                   "single_agent_rollout")
        torch.cuda.synchronize()
        for buf in guards:
            assert bool((buf[:GUARD] == buf[0]).all()) and bool((buf[-GUARD:] == buf[0]).all())
            assert float(buf[0]) == float(SENTINEL[buf.dtype])
        return {k: v.cpu() for k, v in arrays.items()}


def _uniforms(E, seed):
    """[T, E] uniforms in (0, 1] with the edges of the search: 1.0 and values below 1e-8."""
    g = np.random.default_rng(seed)
    u = g.random(T * E).astype(np.float32)
    u[u == 0] = 1.0
    k = np.arange(T * E)
    u[k % 5 == 0] = 1.0
    u[k % 7 == 3] = np.float32(5e-9)
    return torch.from_numpy(u.reshape(T, E)).cuda()


def _ratio(err, bound):
    return float((err / bound).max()) if err.size else 0.0


@pytest.mark.parametrize("case", CASES, ids=[f"{KINDS[c[0]][0]}-{c[5]}-{'x'.join(map(str, c[1]))}"
                                             f"-E{c[2]}-pool{c[3]}-s{c[4]:g}" for c in CASES])
def test_forward_and_selection_within_bound_of_float64(case):
    kind, hidden, E, pool, scale, family = case
    F, A = KINDS[kind][1], KINDS[kind][2]
    layers = R.make_policy([F] + hidden + [A], scale=scale, seed=kind + len(hidden))
    run = Run(kind, E, pool, layers)
    g = torch.Generator(device="cuda").manual_seed(kind)
    if run.continuous:
        noise = {"normals": torch.randn((T, E), device="cuda", generator=g)}
    else:
        noise = {"uniforms": _uniforms(E, kind)}
    a = run.launch(**noise)
    b = run.launch(**noise)
    for k in a:                                 # bit-identical from the same state
        if k != "episodic_reward_sum":          # float atomicAdd: the order of the adds varies
            assert torch.equal(a[k], b[k]), k
    assert int(a["num_completed"][0]) >= E      # post-reset rows are in the batch
    obs = a["obs_batch"].numpy().reshape(T * E, F)
    ref = R.forward(obs, layers, run.continuous, ACTION_SCALE, ACTION_BIAS)
    got = a["probs_batch"].numpy().astype(np.float64).reshape(T * E, -1)
    err = np.abs(got - ref["out"])
    assert (err <= ref["bound"]).all(), _ratio(err, ref["bound"])
    ratio = _ratio(err, ref["bound"])
    acts = a["actions_batch"].numpy().reshape(T * E)
    if run.continuous:
        mean = ref["out"].reshape(T, E)
        want, bound = R.ou_reference(mean, ref["bound"].reshape(T, E), noise["normals"].cpu()
                                     .numpy(), run.init["ou_state"].cpu().numpy().reshape(E),
                                     **OU)
        aerr = np.abs(acts.astype(np.float64) - want.reshape(-1))
        assert (aerr <= bound.reshape(-1)).all(), _ratio(aerr, bound.reshape(-1))
        ratio = max(ratio, _ratio(aerr, bound.reshape(-1)))
    else:
        assert (got[ref["zero"]] == 0).all()
        zeros = int(ref["zero"].sum())
        p32 = a["probs_batch"].numpy().reshape(T * E, A)
        u = noise["uniforms"].cpu().numpy().reshape(-1)
        assert np.array_equal(acts, R.search_index(p32, u))
        idx, decided = R.categorical_float64(ref["out"], ref["bound"], u)
        assert decided.any()
        assert np.array_equal(acts[decided], idx[decided])
        # argmax: first maximum of the recorded row; the float64 argmax where its lead is clear
        c = run.launch(uniforms=noise["uniforms"], use_argmax=True)
        p32 = c["probs_batch"].numpy().reshape(T * E, A)
        ref = R.forward(c["obs_batch"].numpy().reshape(T * E, F), layers)
        err = np.abs(p32.astype(np.float64) - ref["out"])
        assert (err <= ref["bound"]).all(), _ratio(err, ref["bound"])
        acts = c["actions_batch"].numpy().reshape(-1)
        assert np.array_equal(acts, R.argmax_first(p32))
        top, clear = R.argmax_float64(ref["out"], ref["bound"])
        assert clear.any()
        assert np.array_equal(acts[clear], top[clear])
        print(f"\nzero probabilities pinned: {zeros}, rows decided: {decided.mean():.3f}")
    print(f"\nerror/bound {KINDS[kind][0]} {family} {'x'.join(map(str, hidden)) or '-'} "
          f"E={E} scale={scale:g}: {ratio:.3g}")


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_boundary_uniforms_select_like_search_index(kind):
    """Uniforms on the kernel's own float32 CDF values, above its float32 total, at 1.0 and
    below p[0] at the first timestep (whose observation does not depend on the uniforms)."""
    E = 61
    F, A = KINDS[kind][1], KINDS[kind][2]
    layers = R.make_policy([F, 9, 33, A], scale=3.0, seed=5)
    run = Run(kind, E, 0, layers)
    u1 = _uniforms(E, 7)
    first = run.launch(uniforms=u1)
    p0 = first["probs_batch"][0].numpy()
    cdf = np.cumsum(p0, axis=-1, dtype=np.float32)
    u0 = np.empty(E, np.float32)
    for e in range(E):
        j = e % (A + 3)
        if j < A:
            u0[e] = cdf[e, j]                                   # on a CDF value
        elif j == A:
            u0[e] = np.nextafter(cdf[e, -1], np.float32(2))     # above the float32 total
        elif j == A + 1:
            u0[e] = 1.0
        else:
            u0[e] = p0[e, 0] * np.float32(0.5)                  # below p[0]
    u2 = u1.clone()
    u2[0] = torch.from_numpy(u0).cuda()
    second = run.launch(uniforms=u2)
    assert torch.equal(second["probs_batch"][0], first["probs_batch"][0])
    for res, u in ((first, u1), (second, u2)):
        p = res["probs_batch"].numpy().reshape(T * E, A)
        got = res["actions_batch"].numpy().reshape(-1)
        assert np.array_equal(got, R.search_index(p, u.cpu().numpy().reshape(-1)))
    assert np.array_equal(second["actions_batch"][0].numpy(), R.search_index(p0, u0))


def test_malformed_policies_are_refused_without_a_launch():
    """Widths outside 1..64, four hidden layers and, for the discrete kinds, a head whose width
    is not the env's action count (its actions would index past the env's action space)."""
    from warp_drive_b200 import lib as wlib

    L = wlib.load()
    for kind in KINDS:
        F, A = KINDS[kind][1], KINDS[kind][2]
        run = Run(kind, 1, 0, R.make_policy([F, 8, A], seed=1), n_steps=2)
        r, arrays, guards = run.struct()
        # real weights for every variant, so that even a wrong acceptance stays in bounds
        big = torch.zeros(65 * 65, device="cuda")
        uniforms = torch.full((2, 1), 0.5, device="cuda")
        normals = torch.zeros((2, 1), device="cuda")
        r.uniforms, r.normals = wlib.ptr(uniforms), wlib.ptr(normals)

        def variant(dims):
            v = wlib.SaRollout.from_buffer_copy(r)
            v.n_hidden = len(dims) - 2
            for i in range(5):
                v.dims[i] = dims[i] if i < len(dims) and i < 5 else 0
            for i in range(4):
                v.w[i] = v.b[i] = wlib.ptr(big)
            return v

        cases = {"width 65": [F, 65, A], "width 0": [F, 0, A], "four hidden": [F, 8, 8, 8, 8, A]}
        if kind < 3:
            cases.update({"head +1": [F, 8, A + 1], "head -1": [F, 8, A - 1],
                          "head 62": [F, 56, 56, 64, 62]})
        for what, dims in cases.items():
            c0 = wlib.launch_count()
            rc = L.wdb_single_agent_rollout(wlib.stream_ptr(), ctypes.byref(variant(dims)))
            assert rc != 0, (kind, what)
            assert wlib.launch_count() == c0, (kind, what)
        c0 = wlib.launch_count()
        ok = variant([F, 8, A])
        assert L.wdb_single_agent_rollout(wlib.stream_ptr(), ctypes.byref(ok)) == 0, kind
        assert wlib.launch_count() == c0 + 1
        torch.cuda.synchronize()
        for buf in guards:
            assert bool((buf[:GUARD] == buf[0]).all()) and bool((buf[-GUARD:] == buf[0]).all())
