"""Categorical DQN's (C51) host side without a GPU: the float64 reference of one update
(tests/c51_reference.py) against torch autograd through CategoricalDQN and
FullyConnectedCategoricalQ, the projection's mass, the model's refusals, the huber_delta refusal,
the run config, the native pass's and the rollout's shape envelopes, the bindings, the new
kernels' resource use, and the machine code of every earlier kernel of the update and rollout
files."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import c51_reference as ref
import dqn_update_reference as dref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "warp_drive_b200", "csrc")


def _windows(C, EN):
    w = [(s, (5 * s + k) % EN) for s in range(C) for k in range(3)]
    return np.array(w + w[:4], dtype=np.int32)


_DIMS = [[], [8], [6, 7], [5, 7, 9]]


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


def _support(q_net):
    return q_net.support.numpy().astype(np.float64), q_net.delta_z


@pytest.mark.parametrize("weighted", [False, True], ids=["uniform", "weighted"])
@pytest.mark.parametrize("double_q", [True, False], ids=["double_q", "max_target"])
@pytest.mark.parametrize("N", [2, 11, 51])
@pytest.mark.parametrize("n_step,Np", [(1, 1), (1, 3), (3, 1), (3, 3)])
def test_reference_matches_torch_autograd(n_step, Np, N, double_q, weighted):
    from warp_drive_b200.training.algorithms.dqn import CategoricalDQN

    C, E, F, A, gamma = 13, 3, 4, 3, 0.93
    dims = _DIMS[(n_step + Np + N) % 4]
    # a support narrower than the returns: some atom targets clamp at either end
    q_net, target = ref.make_c51_models(F, A, dims, N=N, v_min=-1.5, v_max=2.0,
                                        seed=n_step + 10 * Np + N)
    with torch.no_grad():                      # the target differs from the online network
        for p in target.parameters():
            p.add_(0.3 * torch.randn_like(p))
    ring = dref.make_q_ring(C, E, Np, F, A, seed=n_step + N)
    ring[2][:] *= 2.5                          # rewards past both ends of the support
    windows = _windows(C, E * Np)
    B = len(windows)
    obs, actions, rewards, done, boot_obs = dref.gather(ring, windows, n_step, Np)
    assert (done != 0).any()
    if n_step > 1:                             # a done flag before a window's last step
        assert (done[:-1] != 0).any()
    weights = np.random.default_rng(N).uniform(0.1, 1.0, B) if weighted else None
    z, dz = _support(q_net)
    want = ref.c51_sampled((q_net, target), ring, windows, n_step, gamma, double_q, z, dz,
                           weights)
    tz = want["tz"]
    assert (tz == z[0]).any() and (tz == z[-1]).any()
    assert ((tz > z[0]) & (tz < z[-1])).any()
    # terminal windows: every atom target is the same reward, so all clamp to one end
    term = done[0] != 0
    assert term.any() and np.all(tz[term] == tz[term][:, :1])
    ends = term & ((tz[:, 0] == z[0]) | (tz[:, 0] == z[-1]))
    assert ends.any()
    algo = CategoricalDQN(gamma, n_step=n_step, double_q=double_q)
    q_net.zero_grad()
    loss, qbar, rbar = algo.loss(q_net, target, _t(obs), _t(actions)[:, None], _t(rewards),
                                 _t(done).double(), _t(boot_obs),
                                 weights=None if weights is None else _t(weights))
    loss.backward()
    assert abs(loss.item() - want["loss"]) <= 1e-12
    assert abs(loss.item() * B - want["sum_loss"]) <= 1e-10
    assert np.abs(qbar.numpy() - want["qbar"]).max() <= 1e-12
    assert np.abs(rbar.numpy() - want["rbar"]).max() <= 1e-12
    assert abs(float(qbar.sum()) - want["sum_q"]) <= 1e-10
    names = [n for n, _ in q_net.named_parameters()]
    got = [p.grad.numpy() for p in q_net.parameters()]
    assert len(got) == len(want["grads"]) == 2 * (len(dims) + 1)
    for name, a, b in zip(names, got, want["grads"]):
        assert a.shape == b.shape, name
        assert np.abs(b).max() > 0, name       # every block is reached
        assert np.abs(a - b).max() <= 1e-12, name


def test_projection_conserves_mass():
    g = np.random.default_rng(4)
    N, B = 11, 64
    z = np.arange(N, dtype=np.float64) - 3.0   # dz = 1: atoms and their gaps are exact
    p = ref.softmax(g.standard_normal((B, N)))
    tz = np.clip(g.uniform(-5.0, 9.0, (B, N)), z[0], z[-1])
    tz[:8] = z[g.integers(0, N, (8, N))]       # rows that land exactly on atoms
    m = ref.project(tz, p, z, 1.0)
    assert np.abs(m.sum(axis=1) - p.sum(axis=1)).max() <= 1e-14
    assert np.all(m >= 0)
    # exactly on an atom: all of p'_j goes to it, nothing to its neighbours
    one = ref.project(z[None, [4]], np.ones((1, 1)), z, 1.0)[0]
    assert one[4] == 1.0 and one.sum() == 1.0
    # the model's float32-rounded support: mass kept to its rounding
    q, _ = ref.make_c51_models(4, 2, [8], N=51, v_min=0.0, v_max=100.0)
    zs, dz = _support(q)
    tz = np.clip(g.uniform(-10.0, 110.0, (B, 51)), zs[0], zs[-1])
    p = ref.softmax(g.standard_normal((B, 51)))
    m = ref.project(tz, p, zs, dz)
    assert np.abs(m.sum(axis=1) - 1.0).max() <= 1e-6


def test_support_and_expectation():
    q, _ = ref.make_c51_models(4, 3, [8, 8], N=5, v_min=-1.0, v_max=0.3, seed=2)
    want = (-1.0 + np.arange(5, dtype=np.float64) * (1.3 / 4)).astype(np.float32)
    assert q.support.dtype == torch.float64    # the model was cast; the values stay rounded
    assert np.array_equal(q.support.numpy(), want.astype(np.float64))
    assert q.delta_z == float(np.float32(1.3 / 4))
    assert "support" not in q.state_dict()     # checkpoints hold the parameters only
    obs = torch.randn(7, 4, dtype=torch.float64)
    lg = q.logits(obs)
    assert lg.shape == (7, 3, 5)
    assert torch.equal(lg.reshape(7, 15), q.policy_head(q.trunk(obs)))
    p = q.probabilities(obs)
    assert torch.allclose(p.sum(-1), torch.ones(7, 3, dtype=torch.float64), atol=1e-15)
    qv = q.q_values(obs)
    assert torch.allclose(qv, (p * q.support).sum(-1), rtol=0, atol=0)
    (out,), values = q(obs=obs)
    assert values is None and torch.equal(out, qv)
    assert not hasattr(q, "collapsed_head")


def test_bootstrap_action_is_the_first_argmax_of_the_expectation():
    from warp_drive_b200.training.algorithms.dqn import CategoricalDQN

    q_net, target = ref.make_c51_models(4, 3, [5], N=4, seed=3)
    with torch.no_grad():                      # a tie between actions 0 and 2
        q_net.policy_head.weight.zero_()
        q_net.policy_head.bias.copy_(torch.tensor(
            [1.0, 2.0, 0.0, 0.0, 3.0, 0.0, 0.0, 0.0, 1.0, 2.0, 0.0, 0.0], dtype=torch.float64))
    obs = torch.randn(2, 4, dtype=torch.float64)
    boot = CategoricalDQN(double_q=True).bootstrap_distribution(q_net, target, obs)
    assert torch.equal(boot, target.probabilities(obs)[:, 0])


def test_weighted_loss_with_unit_weights_is_the_uniform_loss():
    from warp_drive_b200.training.algorithms.dqn import CategoricalDQN

    q_net, target = ref.make_c51_models(4, 2, [8, 8], N=7, seed=1)
    ring = dref.make_q_ring(9, 2, 1, 4, 2, seed=1)
    obs, actions, rewards, done, boot_obs = dref.gather(ring, _windows(9, 2), 2, 1)
    args = (q_net, target, _t(obs), _t(actions)[:, None], _t(rewards), _t(done).double(),
            _t(boot_obs))
    algo = CategoricalDQN(0.9, n_step=2)
    a = algo.loss(*args)[0]
    b = algo.loss(*args, weights=torch.ones(len(obs), dtype=torch.float64))[0]
    assert torch.equal(a, b)


def _mk_env(action_space):
    from test_ddpg_update_reference_cpu import _Env

    env = _Env(4, 1)
    env.env.action_space = {0: action_space}
    return env


def test_categorical_model():
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.utils import spaces as sp

    cls = ModelFactory.create("fully_connected_categorical_q")
    q = cls(env=_mk_env(sp.Discrete(3)), model_config={
        "type": "fully_connected_categorical_q", "fc_dims": [8, 6], "v_min": 0, "v_max": 10},
        policy="shared", policy_tag_to_agent_id_map={"shared": [0]})
    assert q.is_q_network and q.is_categorical_q and q.output_dims == [3]
    assert not getattr(q, "is_quantile_q", False)
    assert not getattr(q, "is_implicit_quantile_q", False)
    assert q.num_atoms == 51 and (q.v_min, q.v_max) == (0.0, 10.0)
    assert (q.policy_head.in_features, q.policy_head.out_features) == (6, 153)
    assert [n for n, _ in q.named_parameters()] == [
        "fc.0.0.weight", "fc.0.0.bias", "fc.1.0.weight", "fc.1.0.bias",
        "policy_head.weight", "policy_head.bias"]


def test_categorical_model_refusals():
    from test_ddpg_update_reference_cpu import _Env
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.utils import spaces as sp

    cls = ModelFactory.create("fully_connected_categorical_q")
    qcls = ModelFactory.create("fully_connected_q")
    base = {"type": "fully_connected_categorical_q", "fc_dims": [8], "v_min": -1.0, "v_max": 1.0}
    mk = lambda cfg, space=sp.Discrete(3): cls(  # noqa: E731
        env=_mk_env(space), model_config=dict(base, **cfg),
        policy="shared", policy_tag_to_agent_id_map={"shared": [0]})
    assert mk({"num_atoms": 2}).num_atoms == 2 and mk({"num_atoms": 64}).num_atoms == 64
    for v in (0, 1, 65, 2.0, 8.5, "8", True, None):
        with pytest.raises(ValueError, match="num_atoms"):
            mk({"num_atoms": v})
    for key in ("v_min", "v_max"):
        cfg = dict(base)
        del cfg[key]
        with pytest.raises(ValueError, match=key):
            cls(env=_mk_env(sp.Discrete(3)), model_config=cfg, policy="shared",
                policy_tag_to_agent_id_map={"shared": [0]})
        for v in (float("nan"), float("inf"), -float("inf"), "1", True, None, [1.0]):
            with pytest.raises(ValueError, match=key):
                mk({key: v})
    for lo, hi in ((1.0, 1.0), (2.0, -2.0)):
        with pytest.raises(ValueError, match="v_min < model.v_max"):
            mk({"v_min": lo, "v_max": hi})
    assert mk({"v_min": -3, "v_max": 7}).delta_z == float(np.float32(10 / 50))
    # the refusals of fully_connected_q, with its messages
    qkw = dict(model_config={"type": "fully_connected_q", "fc_dims": [8]}, policy="shared",
               policy_tag_to_agent_id_map={"shared": [0]})
    for space in (sp.Box(-1.0, 1.0, shape=(2,), dtype=np.float32), sp.MultiDiscrete([3, 3]),
                  sp.MultiDiscrete([3])):
        with pytest.raises(ValueError) as want:
            qcls(env=_mk_env(space), **qkw)
        with pytest.raises(ValueError, match="single Discrete") as got:
            mk({}, space)
        assert str(got.value) == str(want.value)
    env = _Env(4, 1)
    env.env.action_space = {0: sp.Discrete(3)}
    env.env.observation_space = {0: sp.Dict({
        "x": sp.Box(-1.0, 1.0, shape=(4,), dtype=np.float32),
        "action_mask": sp.Box(0.0, 1.0, shape=(3,), dtype=np.float32)})}
    with pytest.raises(ValueError) as want:
        qcls(env=env, **qkw)
    with pytest.raises(ValueError, match="action_mask") as got:
        cls(env=env, model_config=base, policy="shared",
            policy_tag_to_agent_id_map={"shared": [0]})
    assert str(got.value) == str(want.value)


def test_c51_run_config_loads():
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_dqn import dqn_policy_settings, epsilon_schedule

    cfg = load_run_config("single_cartpole_c51")
    iqn = load_run_config("single_cartpole_iqn")
    pol, base = cfg["policy"]["shared"], iqn["policy"]["shared"]
    assert pol["algorithm"] == "DQN"
    assert pol["model"] == {"type": "fully_connected_categorical_q", "num_atoms": 51,
                            "v_min": 0, "v_max": 100, "fc_dims": [64, 64],
                            "model_ckpt_filepath": ""}
    assert "huber_delta" not in pol
    assert {k: v for k, v in pol.items() if k != "model"} == {
        k: v for k, v in base.items() if k not in ("model", "huber_delta")}
    assert cfg["trainer"] == iqn["trainer"] and cfg["sampler"] == iqn["sampler"]
    dqn_policy_settings(pol)
    epsilon_schedule(cfg)


def test_categorical_policy_refuses_huber_delta():
    from warp_drive_b200.training.trainer_dqn import categorical_policy_settings

    categorical_policy_settings({"gamma": 0.99})
    for v in (1.0, 2.0, None):
        with pytest.raises(ValueError, match="huber_delta"):
            categorical_policy_settings({"gamma": 0.99, "huber_delta": v})


# ------------------------------------------------------------------------ the native envelope
def _struct(F=4, A=2, dims=(64, 64), N=51, C=100, n_step=3):
    from warp_drive_b200.training.algorithms.dqn import CategoricalDQN
    from warp_drive_b200.training.algorithms.fused_dqn import _shape_struct

    q, _ = ref.make_c51_models(F, A, list(dims), N=N)
    return _shape_struct(CategoricalDQN(0.99, n_step=n_step), q, 8, 1, C)


def _sup(B=256, n_atoms=None, **kw):
    from warp_drive_b200 import lib as wlib

    L = wlib.load()
    u = _struct(**kw)
    n = kw.get("N", 51) if n_atoms is None else n_atoms
    return (L.wdb_c51_update_sampled_supported(ctypes.byref(u), n, B),
            L.wdb_c51_update_sampled_workspace_bytes(ctypes.byref(u), n, B))


def test_supported_checks_the_envelope():
    from qr_dqn_reference import make_qr_models
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.dqn import CategoricalDQN
    from warp_drive_b200.training.algorithms.fused_dqn import fused_c51_supported

    if not os.path.exists(wlib.LIB_PATH):
        pytest.skip("libwdb200.so is not built")
    # the run config's shape: CartPole with [64, 64] and 51 atoms
    assert _sup()[0] == 1 and 0 < _sup(B=16)[1] < _sup(B=4096)[1]
    assert _sup(N=2)[0] == 1 and _sup(N=64)[0] == 1
    assert _sup(n_atoms=1) == (0, -1) and _sup(n_atoms=65) == (0, -1)
    assert _sup(dims=())[0] == 1 and _sup(dims=(64, 64, 64), N=32)[0] == 1
    assert _sup(A=3)[0] == 1                   # MountainCar / Acrobot at the same size
    # shared memory: both networks and the head's gradient block grow with A * N; a third
    # hidden layer of 64 does not fit beside a head of 2 x 51
    assert _sup(dims=(64, 64, 64))[0] == 0 and _sup(dims=(64, 64, 64), A=3, N=64)[0] == 0
    assert _sup(dims=(65,))[0] == 0
    assert _sup(B=0) == (0, -1)
    assert _sup(C=3, n_step=3)[0] == 0 and _sup(C=4, n_step=3)[0] == 1
    assert _sup(F=63)[0] == 1 and _sup(F=64)[0] == 0
    algo = CategoricalDQN(0.99, n_step=3)
    q, _ = ref.make_c51_models(4, 2, [64, 64], N=51)
    assert fused_c51_supported(algo, q.float(), 8, 1, 100, 256) is True
    q, _ = ref.make_c51_models(4, 2, [64, 64, 64, 64], N=51)
    assert fused_c51_supported(algo, q.float(), 8, 1, 100, 256) is False
    qr, _ = make_qr_models(4, 2, 8, [64, 64])
    assert fused_c51_supported(algo, qr.float(), 8, 1, 100, 256) is False


def test_bindings_match_the_header():
    from warp_drive_b200 import lib as wlib

    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    want = {
        "wdb_c51_update_sampled_supported":
            r"int wdb_c51_update_sampled_supported\(const wdb_dqn_update_args \*update, "
            r"int n_atoms,\s+int n_windows\);",
        "wdb_c51_update_sampled_workspace_bytes":
            r"long long wdb_c51_update_sampled_workspace_bytes\(const wdb_dqn_update_args "
            r"\*update,\s+int n_atoms, int n_windows\);",
        "wdb_c51_update_sampled":
            r"int wdb_c51_update_sampled\(void \*stream, const wdb_dqn_update_args \*update, "
            r"int n_atoms,\s+const float \*support, float delta_z,\s+const wdb_replay_windows "
            r"\*windows, const float \*weights\);",
        "wdb_single_agent_rollout_categorical_supported":
            r"int wdb_single_agent_rollout_categorical_supported\(int n_hidden, const int \*dims, "
            r"int n_atoms\);",
    }
    for name, pattern in want.items():
        assert re.search(pattern, header), name
    sig = wlib._SIGNATURES
    dqn = ctypes.POINTER(wlib.DqnUpdate)
    win = ctypes.POINTER(wlib.ReplayWindows)
    assert sig["wdb_c51_update_sampled_supported"] == (ctypes.c_int, [dqn, ctypes.c_int,
                                                                      ctypes.c_int])
    assert sig["wdb_c51_update_sampled_workspace_bytes"] == (
        ctypes.c_longlong, [dqn, ctypes.c_int, ctypes.c_int])
    assert sig["wdb_c51_update_sampled"] == (
        ctypes.c_int, [ctypes.c_void_p, dqn, ctypes.c_int, ctypes.c_void_p, ctypes.c_float, win,
                       ctypes.c_void_p])
    assert sig["wdb_single_agent_rollout_categorical_supported"] == (
        ctypes.c_int, [ctypes.c_int, ctypes.POINTER(ctypes.c_int), ctypes.c_int])


def test_rollout_categorical_predicate():
    from warp_drive_b200 import lib as wlib

    if not os.path.exists(wlib.LIB_PATH):
        pytest.skip("libwdb200.so is not built")
    L = wlib.load()

    def cat(dims, n):
        arr = (ctypes.c_int * 5)(*(list(dims) + [0] * (5 - len(dims))))
        return L.wdb_single_agent_rollout_categorical_supported(len(dims) - 2, arr, n)

    def plain(dims):
        arr = (ctypes.c_int * 5)(*(list(dims) + [0] * (5 - len(dims))))
        return L.wdb_single_agent_rollout_supported(len(dims) - 2, arr)

    # CartPole, [64, 64], 51 atoms: 11 110 floats, under the 11 264-float cap
    assert cat([4, 64, 64, 102], 51) == 1
    assert plain([4, 64, 64, 102]) == 0        # the plain predicate keeps its answer
    # MountainCar and Acrobot at that size do not fit
    assert cat([2, 64, 64, 153], 51) == 0 and cat([6, 64, 64, 153], 51) == 0
    assert cat([2, 32, 32, 153], 51) == 1
    assert cat([4, 64, 64, 102], 1) == 0 and cat([4, 8, 130], 65) == 0
    assert cat([4, 8, 128], 64) == 1 and cat([4, 8, 101], 51) == 0   # A * N
    assert cat([4, 65, 102], 51) == 0 and cat([4, 102], 51) == 1


# ------------------------------------------------------------------------ ptxas / SASS
# The C51 kernels' names contain none of "dqn_pass_kernel", "dqn_weighted_kernel", "qr_dqn_kernel"
# or "iqn", which other tests find kernels by; they live in wdb_c51_update.cu with that file's
# copy of the fixed-order reduction.  The categorical rollout kind is an instantiation of the
# rollout kernel in a file of its own, wdb_sa_rollout_categorical.cu, so wdb_sa_rollout.cu keeps
# its kernel set.
_C51_KERNELS = {
    "10c51_kernelE19wdb_dqn_update_argsNS_4PlanEiPKffPfPdPK4int2",
    "22c51_prioritized_kernelE19wdb_dqn_update_argsNS_4PlanEiPKffPfPdPK4int2S3_",
}
_REDUCE = "18ddpg_reduce_kernelENS_6ReduceEPKfPKdPd"
_SA_CATEGORICAL = "17sa_rollout_kernelILi5EEEv14wdb_sa_rollout"

# The normalised SASS of the IQN kernels, recorded at the parent commit with nvcc 12.9.
_IQN_SASS_SHA256 = {
    "10iqn_kernelE19wdb_dqn_update_args12wdb_iqn_argsNS_4PlanEPfPdPK4int2":
        "dce0926785899c9d33d934f1329842ed5e240dac14a018d18618d95c962129ae",
    "22iqn_prioritized_kernelE19wdb_dqn_update_args12wdb_iqn_argsNS_4PlanEPfPdPK4int2PKf":
        "6a829393aff0b022433301df94bfa42a12fbc978107c596e1eef6a7abc6e0427",
}


def _ptxas(src, tmp_path):
    proc = subprocess.run(
        ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas",
         "-v", "-cubin", "-I", os.path.join(ROOT, "include"), os.path.join(CSRC, src), "-o",
         str(tmp_path / (src + ".cubin"))],
        capture_output=True, text=True, check=True)
    return proc.stderr


def _instructions(cubin):
    """Each kernel's SASS with addresses, the function's own name and the column padding
    dropped."""
    from test_qr_dqn_cpu import _strip

    sass = subprocess.run(["cuobjdump", "-sass", cubin], capture_output=True, text=True,
                          check=True).stdout
    funcs, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = _strip(m.group(1))
            funcs[cur] = []
        elif cur is not None:
            funcs[cur].append(" ".join(re.sub(r"/\*[0-9a-f]{4}\*/", "", line).split()))
    return funcs


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_c51_kernels_compile_without_spills_and_earlier_kernels_keep_their_code(tmp_path):
    from test_qr_dqn_cpu import _KEPT_SASS_SHA256, _cubin, _sass_hashes
    from test_iqn_cpu import _QR_SASS_SHA256

    stats, cubin = _cubin(os.path.join(CSRC, "wdb_c51_update.cu"), tmp_path)
    assert set(stats) == _C51_KERNELS | {_REDUCE}
    for k in _C51_KERNELS:
        assert stats[k]["spill"] == (0, 0), (k, stats[k])
    regs = [int(x) for x in re.findall(r"Used (\d+) registers",
                                       _ptxas("wdb_c51_update.cu", tmp_path))]
    print("C51 kernels' registers (ptxas, sm_90a):", regs)
    assert len(regs) == 3 and all(r <= 255 for r in regs)
    sa_stats, _ = _cubin(os.path.join(CSRC, "wdb_sa_rollout_categorical.cu"), tmp_path)
    assert set(sa_stats) == {_SA_CATEGORICAL}
    assert sa_stats[_SA_CATEGORICAL]["spill"] == (0, 0), sa_stats
    print("categorical rollout:", _ptxas("wdb_sa_rollout_categorical.cu", tmp_path))
    version = subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout
    if "release 12.9" not in version:
        pytest.skip("the recorded SASS is nvcc 12.9's")
    want = dict(_KEPT_SASS_SHA256)
    want["wdb_ddpg_update.cu"] = dict(want["wdb_ddpg_update.cu"], **_QR_SASS_SHA256)
    want["wdb_iqn_update.cu"] = dict(_IQN_SASS_SHA256, **{
        _REDUCE: want["wdb_ddpg_update.cu"][_REDUCE]})
    # the reduction here is the same machine code as the update file's (cuobjdump pads the
    # columns to a file's widest instruction, so the comparison drops the padding)
    _, ddpg_cubin = _cubin(os.path.join(CSRC, "wdb_ddpg_update.cu"), tmp_path)
    assert _instructions(cubin)[_REDUCE] == _instructions(ddpg_cubin)[_REDUCE]
    for src, kept in want.items():
        _, cubin = _cubin(os.path.join(CSRC, src), tmp_path)
        got = _sass_hashes(cubin)
        assert set(got) == set(kept), src      # no kernel lost or added
        assert got == kept, src
