"""Quantile-regression DQN's host side without a GPU: the float64 reference of one update
(tests/qr_dqn_reference.py) against torch autograd through QuantileDQN and
FullyConnectedQuantileQ, the model's refusals, the run config, the native pass's shape envelope,
the new kernels' resource use, and the machine code of every kernel that shares their files."""
import ctypes
import hashlib
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import dqn_update_reference as dref
import qr_dqn_reference as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "warp_drive_b200", "csrc")
NVCC_SM90A = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17"]


def _windows(C, EN):
    w = [(s, (5 * s + k) % EN) for s in range(C) for k in range(3)]
    return np.array(w + w[:4], dtype=np.int32)


_DIMS = [[], [8], [6, 7], [5, 7, 9]]


@pytest.mark.parametrize("weighted", [False, True], ids=["uniform", "weighted"])
@pytest.mark.parametrize("double_q", [True, False], ids=["double_q", "max_target"])
@pytest.mark.parametrize("N", [2, 8, 32])
@pytest.mark.parametrize("n_step,Np", [(1, 1), (1, 3), (3, 1), (3, 3)])
def test_reference_matches_torch_autograd(n_step, Np, N, double_q, weighted):
    from warp_drive_b200.training.algorithms.dqn import QuantileDQN

    C, E, F, A, gamma = 13, 3, 4, 3, 0.93
    dims = _DIMS[(n_step + Np + N) % 4]
    q_net, target = ref.make_qr_models(F, A, N, dims, seed=n_step + 10 * Np + N)
    with torch.no_grad():                      # the target differs from the online network
        for p in target.parameters():
            p.add_(0.3 * torch.randn_like(p))
    ring = dref.make_q_ring(C, E, Np, F, A, seed=n_step + N)
    windows = _windows(C, E * Np)
    B = len(windows)
    obs, actions, rewards, done, boot_obs = dref.gather(ring, windows, n_step, Np)
    assert (done != 0).any()
    if n_step > 1:                             # a done flag before a window's last step
        assert (done[:-1] != 0).any()
    weights = np.random.default_rng(N).uniform(0.1, 1.0, B) if weighted else None
    # kappa at the median |u|: pairs on both sides of the Huber kink
    probe = ref.qr_dqn_sampled((q_net, target), ring, windows, n_step, gamma, 1.0, double_q, N)
    kappa = float(np.median(np.abs(probe["u"])))
    want = ref.qr_dqn_sampled((q_net, target), ring, windows, n_step, gamma, kappa, double_q, N,
                              weights)
    u = want["u"]
    assert (np.abs(u) < kappa).any() and (np.abs(u) > kappa).any()
    assert (u < 0).any() and (u > 0).any()     # both sides of the indicator
    algo = QuantileDQN(gamma, n_step=n_step, double_q=double_q, huber_delta=kappa)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x))  # noqa: E731
    q_net.zero_grad()
    loss, qbar, rbar = algo.loss(q_net, target, t(obs), t(actions)[:, None], t(rewards),
                                 t(done).double(), t(boot_obs),
                                 weights=None if weights is None else t(weights))
    loss.backward()
    assert abs(loss.item() - want["loss"]) <= 1e-12
    assert abs(loss.item() * B - want["sum_loss"]) <= 1e-10
    assert np.abs(qbar.detach().numpy() - want["qbar"]).max() <= 1e-12
    assert np.abs(rbar.numpy() - want["rbar"]).max() <= 1e-12
    assert abs(float(qbar.detach().sum()) - want["sum_q"]) <= 1e-10
    got = [p.grad.numpy() for p in q_net.parameters()]
    assert len(got) == len(want["grads"]) == 2 * (len(dims) + 1)
    for a, b in zip(got, want["grads"]):
        assert a.shape == b.shape
        assert np.abs(a - b).max() <= 1e-12


def test_bootstrap_action_is_the_first_argmax_of_the_mean_quantile():
    from warp_drive_b200.training.algorithms.dqn import QuantileDQN

    q_net, target = ref.make_qr_models(4, 3, 4, [5], seed=3)
    with torch.no_grad():                      # a tie of the means between actions 0 and 2
        q_net.policy_head.weight.zero_()
        q_net.policy_head.bias.copy_(torch.tensor([0, 1, 2, 3, -5, 0, 0, 0, 3, 2, 1, 0.0],
                                                  dtype=torch.float64))
    obs = torch.zeros(2, 4, dtype=torch.float64)
    boot = QuantileDQN(double_q=True).bootstrap_quantiles(q_net, target, obs)
    assert torch.equal(boot, target.quantiles(obs)[:, 0].detach())


def test_weighted_loss_with_unit_weights_is_the_uniform_loss():
    from warp_drive_b200.training.algorithms.dqn import QuantileDQN

    q_net, target = ref.make_qr_models(4, 2, 8, [8, 8], seed=1)
    ring = dref.make_q_ring(9, 2, 1, 4, 2, seed=1)
    obs, actions, rewards, done, boot_obs = dref.gather(ring, _windows(9, 2), 2, 1)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x))  # noqa: E731
    args = (q_net, target, t(obs), t(actions)[:, None], t(rewards), t(done).double(), t(boot_obs))
    algo = QuantileDQN(0.9, n_step=2)
    a = algo.loss(*args)[0]
    b = algo.loss(*args, weights=torch.ones(len(obs), dtype=torch.float64))[0]
    assert torch.equal(a, b)


def test_quantile_model():
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.utils import spaces as sp

    cls = ModelFactory.create("fully_connected_quantile_q")
    q = cls(env=_mk_env(sp.Discrete(3)), model_config={
        "type": "fully_connected_quantile_q", "fc_dims": [8, 8], "num_quantiles": 5},
        policy="shared", policy_tag_to_agent_id_map={"shared": [0]}).double()
    assert q.is_q_network and q.is_quantile_q and q.output_dims == [3]
    assert q.num_quantiles == 5 and q.policy_head.out_features == 15
    assert [n for n, _ in q.named_parameters()] == [
        "fc.0.0.weight", "fc.0.0.bias", "fc.1.0.weight", "fc.1.0.bias",
        "policy_head.weight", "policy_head.bias"]
    obs = torch.randn(2, 7, 4, dtype=torch.float64)
    z = q.policy_head(q.trunk(obs))
    quantiles = q.quantiles(obs)
    assert quantiles.shape == (2, 7, 3, 5)
    for a in range(3):                         # column a * N + i is quantile i of action a
        for i in range(5):
            assert torch.equal(quantiles[..., a, i], z[..., a * 5 + i])
    qv = q.q_values(obs)
    assert qv.shape == (2, 7, 3)
    assert torch.allclose(qv, quantiles.mean(-1), rtol=0, atol=1e-12)
    (out,), values = q(obs=obs)
    assert values is None and torch.equal(out, qv)
    w, b = q.collapsed_head()
    assert torch.equal(w, q.policy_head.weight.view(3, 5, 8).mean(1))
    assert torch.equal(b, q.policy_head.bias.view(3, 5).mean(1))


def test_quantile_model_refusals():
    from test_ddpg_update_reference_cpu import _Env
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.utils import spaces as sp

    cls = ModelFactory.create("fully_connected_quantile_q")
    qcls = ModelFactory.create("fully_connected_q")
    kw = lambda n: dict(  # noqa: E731
        model_config={"type": "fully_connected_quantile_q", "fc_dims": [8], "num_quantiles": n},
        policy="shared", policy_tag_to_agent_id_map={"shared": [0]})
    qkw = dict(model_config={"type": "fully_connected_q", "fc_dims": [8]}, policy="shared",
               policy_tag_to_agent_id_map={"shared": [0]})
    assert cls(env=_mk_env(sp.Discrete(3)), **kw(2)).num_quantiles == 2
    assert cls(env=_mk_env(sp.Discrete(3)), **kw(256)).num_quantiles == 256
    for n in (None, 1, 0, -3, 257, 2.0, 8.5, "8", True):
        with pytest.raises(ValueError, match="num_quantiles"):
            cls(env=_mk_env(sp.Discrete(3)), **kw(n))
    cfg = {"type": "fully_connected_quantile_q", "fc_dims": [8]}
    with pytest.raises(ValueError, match="num_quantiles"):
        cls(env=_mk_env(sp.Discrete(3)), model_config=cfg, policy="shared",
            policy_tag_to_agent_id_map={"shared": [0]})
    # the refusals of fully_connected_q, with its messages
    for space in (sp.Box(-1.0, 1.0, shape=(2,), dtype=np.float32), sp.MultiDiscrete([3, 3]),
                  sp.MultiDiscrete([3])):
        with pytest.raises(ValueError) as want:
            qcls(env=_mk_env(space), **qkw)
        with pytest.raises(ValueError, match="single Discrete") as got:
            cls(env=_mk_env(space), **kw(8))
        assert str(got.value) == str(want.value)
    env = _Env(4, 1)
    env.env.action_space = {0: sp.Discrete(3)}
    env.env.observation_space = {0: sp.Dict({
        "x": sp.Box(-1.0, 1.0, shape=(4,), dtype=np.float32),
        "action_mask": sp.Box(0.0, 1.0, shape=(3,), dtype=np.float32)})}
    with pytest.raises(ValueError) as want:
        qcls(env=env, **qkw)
    with pytest.raises(ValueError, match="action_mask") as got:
        cls(env=env, **kw(8))
    assert str(got.value) == str(want.value)


def _mk_env(action_space):
    from test_ddpg_update_reference_cpu import _Env

    env = _Env(4, 1)
    env.env.action_space = {0: action_space}
    return env


def test_qr_dqn_run_config_loads():
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_dqn import dqn_policy_settings, epsilon_schedule

    cfg = load_run_config("single_cartpole_qr_dqn")
    dqn = load_run_config("single_cartpole_dqn")
    pol, base = cfg["policy"]["shared"], dqn["policy"]["shared"]
    assert pol["algorithm"] == "DQN"
    assert pol["model"] == dict(base["model"], type="fully_connected_quantile_q",
                                num_quantiles=32)
    assert pol["model"]["fc_dims"] == [64, 64]
    assert {k: v for k, v in pol.items() if k != "model"} == {
        k: v for k, v in base.items() if k != "model"}
    assert cfg["trainer"] == dqn["trainer"] and cfg["sampler"] == dqn["sampler"]
    dqn_policy_settings(pol)
    epsilon_schedule(cfg)


def _sup(F=4, A=2, N=8, dims=(64, 64), C=100, n_step=3, B=256, delta=1.0):
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.dqn import QuantileDQN
    from warp_drive_b200.training.algorithms.fused_dqn import _shape_struct

    L = wlib.load()
    q, _ = ref.make_qr_models(F, A, N, list(dims))
    u = _shape_struct(QuantileDQN(0.99, n_step=n_step), q, 8, 1, C)
    u.huber_delta = delta
    return (L.wdb_qr_dqn_update_sampled_supported(ctypes.byref(u), N, B),
            L.wdb_qr_dqn_update_sampled_workspace_bytes(ctypes.byref(u), N, B))


def test_supported_checks_the_envelope():
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.dqn import QuantileDQN
    from warp_drive_b200.training.algorithms.fused_dqn import fused_qr_dqn_supported

    if not os.path.exists(wlib.LIB_PATH):
        pytest.skip("libwdb200.so is not built")
    assert _sup()[0] == 1 and 0 < _sup(B=16)[1] < _sup(B=4096)[1]
    # the head A * N: 64 is taken, 65 and more are not
    for A, N in ((2, 32), (3, 21), (1, 64), (4, 16), (32, 2)):
        assert _sup(A=A, N=N)[0] == 1, (A, N)
    for A, N in ((2, 33), (3, 22), (1, 65), (5, 13), (13, 5)):
        assert _sup(A=A, N=N) == (0, -1), (A, N)
    assert _sup(dims=(64, 64, 64))[0] == 1 and _sup(dims=())[0] == 1
    assert _sup(dims=(65,))[0] == 0
    assert _sup(B=0) == (0, -1)
    assert _sup(C=3, n_step=3)[0] == 0 and _sup(C=4, n_step=3)[0] == 1
    assert _sup(F=63)[0] == 1 and _sup(F=64)[0] == 0
    assert _sup(delta=0.0)[0] == 0
    algo = QuantileDQN(0.99, n_step=3)
    for A, N, want in ((2, 32, True), (2, 33, False), (3, 21, True), (3, 22, False)):
        q, _ = ref.make_qr_models(4, A, N, [64, 64])
        assert fused_qr_dqn_supported(algo, q.float(), 8, 1, 100, 256) is want, (A, N)
    q, _ = dref.make_q_models(4, 2, [64, 64])  # a plain Q network takes the DQN pass
    assert fused_qr_dqn_supported(algo, q.float(), 8, 1, 100, 256) is False


# ------------------------------------------------------------------------ ptxas / SASS
def _cubin(src, tmp_path):
    out = str(tmp_path / (os.path.basename(src) + ".cubin"))
    proc = subprocess.run(NVCC_SM90A + ["-Xptxas", "-v", "-cubin", "-I",
                                        os.path.join(ROOT, "include"), src, "-o", out],
                          capture_output=True, text=True, check=True)
    stats, name = {}, None
    for line in proc.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name = _strip(m.group(1))
            stats[name] = {}
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name and "spill" not in stats[name]:
            stats[name]["spill"] = (int(m.group(1)), int(m.group(2)))
    return stats, out


def _strip(name):
    """A kernel's mangled name without its file's anonymous-namespace prefix."""
    return re.sub(r"^_ZN\d+_GLOBAL__N__\w+?_cu_[0-9a-f]{8}", "", name)


def _sass_hashes(cubin):
    """Normalised SASS (addresses and the function's own name dropped) of every kernel."""
    sass = subprocess.run(["cuobjdump", "-sass", cubin], capture_output=True, text=True,
                          check=True).stdout
    funcs, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = _strip(m.group(1))
            assert cur not in funcs, cur
            funcs[cur] = []
        elif cur is not None:
            funcs[cur].append(re.sub(r"/\*[0-9a-f]{4}\*/", "", line).rstrip())
    return {k: hashlib.sha256("\n".join(v).encode()).hexdigest() for k, v in funcs.items()}


# Their names contain neither "dqn_pass_kernel" nor "dqn_weighted_kernel", which find DQN's
# kernels by substring.
_QR_KERNELS = {
    "13qr_dqn_kernelE19wdb_dqn_update_argsNS_4PlanEiPfPdPK4int2",
    "25qr_dqn_prioritized_kernelE19wdb_dqn_update_argsNS_4PlanEiPfPdPK4int2PKf",
}

# The normalised SASS of every kernel of the two files before QR-DQN joined them, recorded at
# the parent commit with nvcc 12.9.
_KEPT_SASS_SHA256 = {
    "wdb_ddpg_update.cu": {
        "15dqn_pass_kernelE19wdb_dqn_update_argsNS_4PlanEPfPdPK4int2":
            "6ddc90ace4fb4f4e215234478611c5493c6e854d826da4ab2c899380da37d283",
        "19dqn_weighted_kernelE19wdb_dqn_update_argsNS_4PlanEPfPdPK4int2PKf":
            "dc12cef1c072dd3daa2b9d2b24c204cef2149407bb4c97cefe5fae82035f2541",
        "16sac_actor_kernelINS_9NoWindowsEEEv19wdb_sac_update_argsNS_4PlanEPfPdT_":
            "5e3dddfb3ee486667e1c9cc52d3fe31e7c70a2445be11b4e0f8cf8ecd3766537",
        "16sac_actor_kernelIPK4int2EEv19wdb_sac_update_argsNS_4PlanEPfPdT_":
            "86bea485eed4957d8e592ffcd6888de1976c8e612d9d2266a7242acea2184237",
        "16td3_actor_kernelINS_9NoWindowsEEEv19wdb_td3_update_argsNS_4PlanEPfPdT_":
            "baa1f44c5fde6671d02a45f1973dd31e95d8d52b2cd29ad6f81c106bc5a9b612",
        "16td3_actor_kernelIPK4int2EEv19wdb_td3_update_argsNS_4PlanEPfPdT_":
            "785909197a2abef31f4c2f8fdaf922101bf73d455fe421dbc2377bea8ab4a388",
        "17sac_critic_kernelINS_9NoWindowsEEEv19wdb_sac_update_argsNS_4PlanEPfPdT_":
            "e963a0aa5bfe088ed0ac0b725bf126499d2386a18edfda269dd6c9078dbb4266",
        "17sac_critic_kernelIPK4int2EEv19wdb_sac_update_argsNS_4PlanEPfPdT_":
            "cc8270109477b67b20fd7165e43fee4063342aa9dc811c221db428abad943258",
        "17td3_critic_kernelINS_9NoWindowsEEEv19wdb_td3_update_argsNS_4PlanEPfPdT_":
            "9ea51c60bf071869f36de6c0668b280a7dc51dc454cd5abd4af04307c46f3ac4",
        "17td3_critic_kernelIPK4int2EEv19wdb_td3_update_argsNS_4PlanEPfPdT_":
            "bdb79e4a2a1926b5d2a56d689ceae355645d294d6a67bbf9c564d66a1b5a73bb",
        "18ddpg_reduce_kernelENS_6ReduceEPKfPKdPd":
            "4ad80efbdf62dead0279d0872ad06dadfc625476fb41c2e1bf18b8292e280def",
        "18ddpg_update_kernelINS_9NoWindowsEEEv20wdb_ddpg_update_argsNS_4PlanEPfPdT_":
            "43727eb73fb299e5ca72c15d364be91aa0dc4bb253d8bcd24a5d3ef3d3cdd04f",
        "18ddpg_update_kernelIPK4int2EEv20wdb_ddpg_update_argsNS_4PlanEPfPdT_":
            "3c1bc0aad87b8df9296a4e1b260f6561df0e407bc08c6a97ac4f681cd717437e",
    },
    "wdb_sa_rollout.cu": {
        "17sa_rollout_kernelILi0EEEv14wdb_sa_rollout":
            "281b4fbcb8b090b3c004a7177d116ce01d9f7eccf7464bf76181381d465fcdc4",
        "17sa_rollout_kernelILi1EEEv14wdb_sa_rollout":
            "e9440085d721d2e49daea49ee9cadf190d1c7a71770c05d72b8550214242d2d5",
        "17sa_rollout_kernelILi2EEEv14wdb_sa_rollout":
            "416864e0a61a02291bba8789103b3352cd9a4d1eb33bf5297b197f921bb73080",
        "17sa_rollout_kernelILi3EEEv14wdb_sa_rollout":
            "15f98aac6ee960bab86a90d2984920c80878eca8981a11e29e51fabcd9b66047",
        "17sa_rollout_kernelILi4EEEv14wdb_sa_rollout":
            "39540458924f10a1f08793008c094a32b6e6a06442c5c028afc661655b7c131b",
    },
}


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_qr_dqn_kernels_compile_without_spills_and_existing_kernels_keep_their_code(tmp_path):
    stats, cubin = _cubin(os.path.join(CSRC, "wdb_ddpg_update.cu"), tmp_path)
    for k in _QR_KERNELS:
        assert stats[k]["spill"] == (0, 0), (k, stats[k])
    version = subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout
    if "release 12.9" not in version:
        pytest.skip("the recorded SASS is nvcc 12.9's")
    for src, want in _KEPT_SASS_SHA256.items():
        if src != "wdb_ddpg_update.cu":
            _, cubin = _cubin(os.path.join(CSRC, src), tmp_path)
        got = _sass_hashes(cubin)
        new = _QR_KERNELS if src == "wdb_ddpg_update.cu" else set()
        assert set(got) == set(want) | new, src       # no kernel lost, only the new ones added
        assert {k: got[k] for k in want} == want, src
