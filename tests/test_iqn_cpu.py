"""Implicit quantile networks' host side without a GPU: the float64 reference of one update
(tests/iqn_reference.py) against torch autograd through ImplicitQuantileDQN and
FullyConnectedIQN, the collapsed head, the model's refusals, the run config, the native pass's
shape envelope and argument struct, the new kernels' resource use, and the machine code of every
earlier kernel of the update and rollout files."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import dqn_update_reference as dref
import iqn_reference as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "warp_drive_b200", "csrc")


def _windows(C, EN):
    w = [(s, (5 * s + k) % EN) for s in range(C) for k in range(3)]
    return np.array(w + w[:4], dtype=np.int32)


_DIMS = [[5], [6, 7], [5, 7, 9]]


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


@pytest.mark.parametrize("weighted", [False, True], ids=["uniform", "weighted"])
@pytest.mark.parametrize("double_q", [True, False], ids=["double_q", "max_target"])
@pytest.mark.parametrize("n_step,Np", [(1, 1), (1, 2), (3, 1), (3, 2)])
def test_reference_matches_torch_autograd(n_step, Np, double_q, weighted):
    from warp_drive_b200.training.algorithms.dqn import ImplicitQuantileDQN

    C, E, F, A, gamma = 13, 3, 4, 3, 0.93
    dims = _DIMS[(n_step + Np) % 3]
    N, NP = 4 + n_step, 3 + 2 * Np
    q_net, target = ref.make_iqn_models(F, A, dims, n_cos=6, N=N, NP=NP, K=5,
                                        seed=n_step + 10 * Np)
    with torch.no_grad():                      # the target differs from the online network
        for p in target.parameters():
            p.add_(0.3 * torch.randn_like(p))
        for net in (q_net, target):            # no head bias for a* to follow, and most
            net.policy_head.bias.zero_()       # embedding units active
            net.tau_embedding.bias.add_(0.5)
    ring = dref.make_q_ring(C, E, Np, F, A, seed=n_step + Np)
    windows = _windows(C, E * Np)
    B = len(windows)
    obs, actions, rewards, done, boot_obs = dref.gather(ring, windows, n_step, Np)
    assert (done != 0).any()
    if n_step > 1:                             # a done flag before a window's last step
        assert (done[:-1] != 0).any()
    g = np.random.default_rng(n_step + Np)
    taus = g.uniform(0.0, 1.0, (B, N + NP))
    weights = g.uniform(0.1, 1.0, B) if weighted else None
    # kappa at the median |u|: pairs on both sides of the Huber kink
    probe = ref.iqn_sampled((q_net, target), ring, windows, n_step, gamma, 1.0, double_q, taus)
    kappa = float(np.median(np.abs(probe["u"])))
    want = ref.iqn_sampled((q_net, target), ring, windows, n_step, gamma, kappa, double_q, taus,
                           weights)
    u = want["u"]
    assert (np.abs(u) < kappa).any() and (np.abs(u) > kappa).any()
    assert (u < 0).any() and (u > 0).any()     # both sides of the indicator
    algo = ImplicitQuantileDQN(gamma, n_step=n_step, double_q=double_q, huber_delta=kappa)
    q_net.zero_grad()
    loss, qbar, rbar = algo.loss(q_net, target, _t(obs), _t(actions)[:, None], _t(rewards),
                                 _t(done).double(), _t(boot_obs),
                                 weights=None if weights is None else _t(weights), taus=_t(taus))
    loss.backward()
    assert abs(loss.item() - want["loss"]) <= 1e-12
    assert abs(loss.item() * B - want["sum_loss"]) <= 1e-10
    assert np.abs(qbar.detach().numpy() - want["qbar"]).max() <= 1e-12
    assert np.abs(rbar.numpy() - want["rbar"]).max() <= 1e-12
    assert abs(float(qbar.detach().sum()) - want["sum_q"]) <= 1e-10
    names = [n for n, _ in q_net.named_parameters()]
    got = [p.grad.numpy() for p in q_net.parameters()]
    assert len(got) == len(want["grads"]) == 2 * (len(dims) + 2)
    assert names[-4:] == ["policy_head.weight", "policy_head.bias", "tau_embedding.weight",
                          "tau_embedding.bias"]
    for name, a, b in zip(names, got, want["grads"]):
        assert a.shape == b.shape, name
        assert np.abs(b).max() > 0, name       # every block is reached
        assert np.abs(a - b).max() <= 1e-12, name


def test_q_values_are_the_mean_over_the_midpoints():
    q, _ = ref.make_iqn_models(4, 3, [8, 8], n_cos=7, K=9, seed=2)
    obs = torch.randn(11, 4, dtype=torch.float64)
    levels = q.acting_levels()
    assert torch.equal(levels, torch.tensor(ref.midpoints(9)))
    z = q.quantiles_at(obs, levels)
    assert z.shape == (11, 9, 3)
    qv = q.q_values(obs)
    assert torch.allclose(qv, z.mean(dim=1), rtol=0, atol=1e-12)
    (out,), values = q(obs=obs)
    assert values is None and torch.equal(out, qv)
    w, b = q.collapsed_head()                  # (W diag(c-bar), b)
    cbar = q.embedding(levels).mean(0)
    assert torch.equal(w, q.policy_head.weight * cbar) and torch.equal(b, q.policy_head.bias)
    # per-row levels [B, T] and shared ones [T] agree
    per_row = q.quantiles_at(obs, levels.expand(11, 9))
    assert torch.allclose(per_row, z, rtol=0, atol=1e-12)
    # the constant feature i = 0 and the cosine ones
    cf = q.cos_features(torch.tensor([0.25], dtype=torch.float64))
    assert torch.allclose(cf[0], torch.cos(torch.pi * torch.arange(7.0, dtype=torch.float64)
                                           * 0.25), rtol=0, atol=1e-15)
    assert cf[0, 0] == 1.0


def test_bootstrap_action_is_the_first_argmax_of_the_collapsed_head():
    from warp_drive_b200.training.algorithms.dqn import ImplicitQuantileDQN

    q_net, target = ref.make_iqn_models(4, 3, [5], seed=3)
    with torch.no_grad():                      # a tie between actions 0 and 2
        q_net.policy_head.weight.zero_()
        q_net.policy_head.bias.copy_(torch.tensor([2.0, -1.0, 2.0], dtype=torch.float64))
    obs = torch.randn(2, 4, dtype=torch.float64)
    taus = torch.rand(2, 5, dtype=torch.float64)
    boot = ImplicitQuantileDQN(double_q=True).bootstrap_quantiles(q_net, target, obs, taus)
    assert torch.equal(boot, target.quantiles_at(obs, taus)[..., 0])


def test_weighted_loss_with_unit_weights_is_the_uniform_loss():
    from warp_drive_b200.training.algorithms.dqn import ImplicitQuantileDQN

    q_net, target = ref.make_iqn_models(4, 2, [8, 8], seed=1)
    ring = dref.make_q_ring(9, 2, 1, 4, 2, seed=1)
    obs, actions, rewards, done, boot_obs = dref.gather(ring, _windows(9, 2), 2, 1)
    taus = torch.rand(len(obs), 9, dtype=torch.float64)
    args = (q_net, target, _t(obs), _t(actions)[:, None], _t(rewards), _t(done).double(),
            _t(boot_obs))
    algo = ImplicitQuantileDQN(0.9, n_step=2)
    a = algo.loss(*args, taus=taus)[0]
    b = algo.loss(*args, weights=torch.ones(len(obs), dtype=torch.float64), taus=taus)[0]
    assert torch.equal(a, b)


def _mk_env(action_space):
    from test_ddpg_update_reference_cpu import _Env

    env = _Env(4, 1)
    env.env.action_space = {0: action_space}
    return env


def test_iqn_model():
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.utils import spaces as sp

    cls = ModelFactory.create("fully_connected_iqn")
    q = cls(env=_mk_env(sp.Discrete(3)), model_config={
        "type": "fully_connected_iqn", "fc_dims": [8, 6]},
        policy="shared", policy_tag_to_agent_id_map={"shared": [0]})
    assert q.is_q_network and q.is_implicit_quantile_q and q.output_dims == [3]
    assert not getattr(q, "is_quantile_q", False)
    assert (q.num_cosines, q.num_tau_samples, q.num_tau_prime_samples,
            q.num_quantile_samples) == (64, 32, 32, 32)
    assert (q.tau_embedding.in_features, q.tau_embedding.out_features) == (64, 6)
    assert (q.policy_head.in_features, q.policy_head.out_features) == (6, 3)
    assert [n for n, _ in q.named_parameters()] == [
        "fc.0.0.weight", "fc.0.0.bias", "fc.1.0.weight", "fc.1.0.bias",
        "policy_head.weight", "policy_head.bias", "tau_embedding.weight", "tau_embedding.bias"]


def test_iqn_model_refusals():
    from test_ddpg_update_reference_cpu import _Env
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.utils import spaces as sp

    cls = ModelFactory.create("fully_connected_iqn")
    qcls = ModelFactory.create("fully_connected_q")
    mk = lambda cfg, space=sp.Discrete(3): cls(  # noqa: E731
        env=_mk_env(space), model_config=dict({"type": "fully_connected_iqn"}, **cfg),
        policy="shared", policy_tag_to_agent_id_map={"shared": [0]})
    for dims in ({}, {"fc_dims": []}, {"fc_dims": None}):
        with pytest.raises(ValueError, match="fc_dims"):
            mk(dims)
    for key, top in (("num_cosines", 64), ("num_tau_samples", 64),
                     ("num_tau_prime_samples", 64), ("num_quantile_samples", 256)):
        assert getattr(mk({"fc_dims": [8], key: 1}), key) == 1
        assert getattr(mk({"fc_dims": [8], key: top}), key) == top
        for v in (0, -2, top + 1, 2.0, 8.5, "8", True, False, None):
            with pytest.raises(ValueError, match=key):
                mk({"fc_dims": [8], key: v})
    # the refusals of fully_connected_q, with its messages
    qkw = dict(model_config={"type": "fully_connected_q", "fc_dims": [8]}, policy="shared",
               policy_tag_to_agent_id_map={"shared": [0]})
    for space in (sp.Box(-1.0, 1.0, shape=(2,), dtype=np.float32), sp.MultiDiscrete([3, 3]),
                  sp.MultiDiscrete([3])):
        with pytest.raises(ValueError) as want:
            qcls(env=_mk_env(space), **qkw)
        with pytest.raises(ValueError, match="single Discrete") as got:
            mk({"fc_dims": [8]}, space)
        assert str(got.value) == str(want.value)
    env = _Env(4, 1)
    env.env.action_space = {0: sp.Discrete(3)}
    env.env.observation_space = {0: sp.Dict({
        "x": sp.Box(-1.0, 1.0, shape=(4,), dtype=np.float32),
        "action_mask": sp.Box(0.0, 1.0, shape=(3,), dtype=np.float32)})}
    with pytest.raises(ValueError) as want:
        qcls(env=env, **qkw)
    with pytest.raises(ValueError, match="action_mask") as got:
        cls(env=env, model_config={"type": "fully_connected_iqn", "fc_dims": [8]},
            policy="shared", policy_tag_to_agent_id_map={"shared": [0]})
    assert str(got.value) == str(want.value)


def test_iqn_run_config_loads():
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_dqn import dqn_policy_settings, epsilon_schedule

    cfg = load_run_config("single_cartpole_iqn")
    qr = load_run_config("single_cartpole_qr_dqn")
    pol, base = cfg["policy"]["shared"], qr["policy"]["shared"]
    assert pol["algorithm"] == "DQN"
    want = {k: v for k, v in base["model"].items() if k != "num_quantiles"}
    assert pol["model"] == dict(want, type="fully_connected_iqn", num_cosines=64,
                                num_tau_samples=32, num_tau_prime_samples=32,
                                num_quantile_samples=32)
    assert pol["model"]["fc_dims"] == [64, 64]
    assert {k: v for k, v in pol.items() if k != "model"} == {
        k: v for k, v in base.items() if k != "model"}
    assert cfg["trainer"] == qr["trainer"] and cfg["sampler"] == qr["sampler"]
    dqn_policy_settings(pol)
    epsilon_schedule(cfg)


# ------------------------------------------------------------------------ the native envelope
def _structs(F=4, A=2, dims=(64, 64), n_cos=64, N=32, NP=32, K=32, C=100, n_step=3, delta=1.0):
    from warp_drive_b200.training.algorithms.dqn import ImplicitQuantileDQN
    from warp_drive_b200.training.algorithms.fused_dqn import _iqn_struct, _shape_struct

    q, _ = ref.make_iqn_models(F, A, list(dims), n_cos=n_cos, N=N, NP=NP, K=K)
    u = _shape_struct(ImplicitQuantileDQN(0.99, n_step=n_step), q, 8, 1, C)
    u.huber_delta = delta
    return u, _iqn_struct(q)


def _sup(B=256, fields=None, **kw):
    """(_supported, _workspace_bytes) of a shape; fields: values written into wdb_iqn_args
    past what the model takes."""
    from warp_drive_b200 import lib as wlib

    L = wlib.load()
    u, a = _structs(**kw)
    for k, v in (fields or {}).items():
        setattr(a, k, v)
    return (L.wdb_iqn_update_sampled_supported(ctypes.byref(u), ctypes.byref(a), B),
            L.wdb_iqn_update_sampled_workspace_bytes(ctypes.byref(u), ctypes.byref(a), B))


def test_supported_checks_the_envelope():
    from qr_dqn_reference import make_qr_models
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.dqn import ImplicitQuantileDQN
    from warp_drive_b200.training.algorithms.fused_dqn import fused_iqn_supported

    if not os.path.exists(wlib.LIB_PATH):
        pytest.skip("libwdb200.so is not built")
    assert _sup()[0] == 1 and 0 < _sup(B=16)[1] < _sup(B=4096)[1]
    # the run config's shape with a third hidden layer of 64, and every count at its largest;
    # shared memory runs out for three layers of 64 with n_cos = 64 and A = 32 (two take A = 64)
    assert _sup(dims=(64, 64, 64), N=64, NP=64, K=256)[0] == 1
    assert _sup(dims=(64, 64, 64), A=16)[0] == 1 and _sup(dims=(64, 64, 64), A=32)[0] == 0
    assert _sup(dims=(64, 64), A=64)[0] == 1
    assert _sup(dims=(1,), n_cos=1, N=1, NP=1, K=1, A=1, F=1)[0] == 1
    for key, field, top in (("n_cos", "n_cos", 64), ("N", "n_tau", 64),
                            ("NP", "n_tau_prime", 64), ("K", "n_quantile_samples", 256)):
        assert _sup(**{key: top})[0] == 1, key
        assert _sup(fields={field: top + 1}) == (0, -1), key
        assert _sup(fields={field: 0}) == (0, -1), key
    assert _sup(dims=(65,))[0] == 0
    assert _sup(A=64)[0] == 1 and _sup(A=65)[0] == 0
    assert _sup(B=0) == (0, -1)
    assert _sup(C=3, n_step=3)[0] == 0 and _sup(C=4, n_step=3)[0] == 1
    assert _sup(F=63)[0] == 1 and _sup(F=64)[0] == 0
    assert _sup(delta=0.0)[0] == 0
    # no hidden layer: nothing for the embedding to multiply (the model refuses it too)
    u, a = _structs()
    u.q.n_hidden = u.target_q.n_hidden = 0
    assert wlib.load().wdb_iqn_update_sampled_supported(ctypes.byref(u), ctypes.byref(a), 8) == 0
    algo = ImplicitQuantileDQN(0.99, n_step=3)
    q, _ = ref.make_iqn_models(4, 2, [64, 64], n_cos=64, N=32, NP=32, K=32)
    assert fused_iqn_supported(algo, q.float(), 8, 1, 100, 256) is True
    q, _ = ref.make_iqn_models(4, 2, [64, 64, 64, 64], n_cos=64)
    assert fused_iqn_supported(algo, q.float(), 8, 1, 100, 256) is False
    qr, _ = make_qr_models(4, 2, 8, [64, 64])
    assert fused_iqn_supported(algo, qr.float(), 8, 1, 100, 256) is False


def test_iqn_args_layout_matches_the_header(tmp_path):
    from test_abi_layout_cpu import _c_fields
    from warp_drive_b200 import lib as wlib

    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    fields = _c_fields(header, "wdb_iqn_args")
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "wdb200.h"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(wdb_iqn_args));']
    lines += [f'  printf("{f} %zu\\n", offsetof(wdb_iqn_args, {f}));' for f in fields]
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)],
                   check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    got = dict((k, int(v)) for k, v in (line.split() for line in out.splitlines()))
    assert ctypes.sizeof(wlib.IqnArgs) == got["size"]
    assert [n for n, _ in wlib.IqnArgs._fields_] == fields
    for f in fields:
        assert getattr(wlib.IqnArgs, f).offset == got[f], f


# ------------------------------------------------------------------------ ptxas / SASS
# The IQN kernels' names contain none of "dqn_pass_kernel", "dqn_weighted_kernel" or "qr_dqn",
# which other tests find kernels by; they live in wdb_iqn_update.cu with that file's copy of
# the fixed-order reduction.
_IQN_KERNELS = {
    "10iqn_kernelE19wdb_dqn_update_args12wdb_iqn_argsNS_4PlanEPfPdPK4int2",
    "22iqn_prioritized_kernelE19wdb_dqn_update_args12wdb_iqn_argsNS_4PlanEPfPdPK4int2PKf",
}
_REDUCE = "18ddpg_reduce_kernelENS_6ReduceEPKfPKdPd"

# The normalised SASS of every kernel of the two files before IQN, recorded at the parent commit
# with nvcc 12.9: the QR-DQN kernels beside the ones tests/test_qr_dqn_cpu.py pins.
_QR_SASS_SHA256 = {
    "13qr_dqn_kernelE19wdb_dqn_update_argsNS_4PlanEiPfPdPK4int2":
        "f1c51c9b56ce470387e659fc734792abfa0296494785e954af839543ac699eca",
    "25qr_dqn_prioritized_kernelE19wdb_dqn_update_argsNS_4PlanEiPfPdPK4int2PKf":
        "b946ed57d43d578939dd477445f7758caefd27a31299819fe4b841165865c1c5",
}


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_iqn_kernels_compile_without_spills_and_earlier_kernels_keep_their_code(tmp_path):
    from test_qr_dqn_cpu import _KEPT_SASS_SHA256, _cubin, _sass_hashes

    stats, cubin = _cubin(os.path.join(CSRC, "wdb_iqn_update.cu"), tmp_path)
    assert set(stats) == _IQN_KERNELS | {_REDUCE}
    for k in _IQN_KERNELS:
        assert stats[k]["spill"] == (0, 0), (k, stats[k])
    proc = subprocess.run(
        ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas",
         "-v", "-cubin", "-I", os.path.join(ROOT, "include"),
         os.path.join(CSRC, "wdb_iqn_update.cu"), "-o", str(tmp_path / "r.cubin")],
        capture_output=True, text=True, check=True)
    regs = [int(x) for x in re.findall(r"Used (\d+) registers", proc.stderr)]
    print("IQN kernels' registers (ptxas, sm_90a):", regs)
    assert len(regs) == 3 and all(r <= 255 for r in regs)
    version = subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout
    if "release 12.9" not in version:
        pytest.skip("the recorded SASS is nvcc 12.9's")
    iqn = _sass_hashes(cubin)
    want = dict(_KEPT_SASS_SHA256)
    want["wdb_ddpg_update.cu"] = dict(want["wdb_ddpg_update.cu"], **_QR_SASS_SHA256)
    # the reduction here is the same machine code as the update file's
    assert iqn[_REDUCE] == want["wdb_ddpg_update.cu"][_REDUCE]
    for src, kept in want.items():
        _, cubin = _cubin(os.path.join(CSRC, src), tmp_path)
        got = _sass_hashes(cubin)
        assert set(got) == set(kept), src      # no kernel lost or added
        assert got == kept, src
