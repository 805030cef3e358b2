"""Branching DQN without a GPU: the float64 reference (tests/branching_q_reference.py) against
torch autograd through BranchingDQN.loss, the branching Q model and its refusals, the native
pass selection, the struct and bindings against the header, the pass's envelope, and what
ptxas makes of the new translation unit."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import branching_q_reference as bref
from dqn_update_reference import dqn_sampled, make_q_models
from test_ddpg_update_reference_cpu import _Env

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "warp_drive_b200", "csrc")
NVCC_SM90A = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC"]


def _lib_or_skip():
    from warp_drive_b200 import lib as wlib

    if not os.path.exists(wlib.LIB_PATH):
        pytest.skip("libwdb200.so is not built")
    return wlib


def _windows(C, E, Np, n_step, B, seed):
    g = np.random.default_rng(seed)
    return np.stack([g.integers(0, C - n_step, B), g.integers(0, E * Np, B)], 1).astype(np.int32)


def _torch_update(models, ring, windows, n_step, gamma, delta, double_q, weights=None):
    from warp_drive_b200.training.algorithms.dqn import BranchingDQN

    q_net, target = models
    Np = ring[0].shape[2]
    obs, actions, rewards, done, boot_obs = (
        torch.from_numpy(np.asarray(x)) for x in bref.gather_branching(ring, windows, n_step, Np))
    algo = BranchingDQN(gamma, n_step=n_step, double_q=double_q, huber_delta=delta)
    q_net.zero_grad()
    w = None if weights is None else torch.from_numpy(weights)
    loss, q, R = algo.loss(q_net, target, obs, actions, rewards, done.double(), boot_obs, w)
    loss.backward()
    grads = [p.grad.numpy() for p in q_net.parameters()]
    return float(loss), q.detach().numpy(), R.numpy(), grads


# (sizes, fc_dims, double_q, n_step, Np, weighted)
_CASES = [
    ([3], [8], True, 1, 1, False),
    ([3], [8, 8], False, 3, 2, True),
    ([5, 3], [16], True, 3, 2, False),
    ([5, 3], [16], False, 1, 1, True),
    ([2, 7, 4], [], True, 3, 3, True),
    ([2, 7, 4], [8, 8, 8], False, 3, 1, False),
    ([21, 21], [16, 16], True, 3, 2, True),
]


@pytest.mark.parametrize("case", range(len(_CASES)))
def test_reference_matches_torch_autograd_in_float64(case):
    sizes, dims, double_q, n_step, Np, weighted = _CASES[case]
    F, C, E, B = 5, 12, 3, 40
    models = bref.make_branching_models(F, sizes, dims, seed=case)
    ring = bref.make_branching_ring(C, E, Np, F, sizes, seed=case)
    windows = _windows(C, E, Np, n_step, B, case)
    weights = (np.random.default_rng(case).uniform(0.2, 1.5, B) if weighted else None)
    ref = bref.branching_sampled(models, ring, windows, n_step, 0.9, 0.7, double_q, sizes,
                                 weights)
    loss, q, R, grads = _torch_update(models, ring, windows, n_step, 0.9, 0.7, double_q, weights)
    assert abs(loss - ref["loss"]) <= 1e-12 * max(1.0, abs(loss))
    np.testing.assert_allclose(q, ref["q"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(R, ref["returns"], rtol=1e-12, atol=1e-12)
    for g, want in zip(grads, ref["grads"]):
        np.testing.assert_allclose(g, want, rtol=1e-12, atol=1e-12)


def test_ties_take_each_heads_first_maximum():
    """Two columns of every head tie in the online network on every obs' (equal rows, and a
    bias that makes them the head's maximum) while the target tells them apart: the double-Q
    bootstrap must read the target at each head's first maximum, in torch and the reference."""
    sizes, F, C, E, Np, n_step, B = [3, 4], 4, 10, 2, 1, 2, 32
    models = bref.make_branching_models(F, sizes, [8], seed=7)
    with torch.no_grad():
        W, b = models[0].policy_head.weight, models[0].policy_head.bias
        for o in bref.offsets(sizes):
            W[o + 1] = W[o]
            b[o] = b[o + 1] = 50.0
            models[1].policy_head.bias[o + 1] = models[1].policy_head.bias[o] + 3.0
    ring = bref.make_branching_ring(C, E, Np, F, sizes, seed=3)
    windows = _windows(C, E, Np, n_step, B, 3)
    ref = bref.branching_sampled(models, ring, windows, n_step, 0.9, 1.0, True, sizes)
    _, _, R, _ = _torch_update(models, ring, windows, n_step, 0.9, 1.0, True)
    np.testing.assert_allclose(R, ref["returns"], rtol=1e-12, atol=1e-12)
    boot_obs = torch.from_numpy(bref.gather_branching(ring, windows, n_step, Np)[4])
    qt = models[1].q_values(boot_obs).detach().numpy()
    want = np.mean([qt[:, o] for o in bref.offsets(sizes)], axis=0)
    np.testing.assert_allclose(ref["boot"], want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("double_q", [True, False])
def test_one_head_is_dqn(double_q):
    """At D = 1 the branching objective is DQN's: same seed, same weights, same update."""
    F, A, C, E, Np, n_step, B = 4, 5, 10, 2, 2, 3, 24
    branching = bref.make_branching_models(F, [A], [8, 8], seed=4)
    plain = make_q_models(F, A, [8, 8], seed=4)
    for a, b in zip(branching[0].parameters(), plain[0].parameters()):
        assert torch.equal(a, b)
    ring = bref.make_branching_ring(C, E, Np, F, [A], seed=5)
    windows = _windows(C, E, Np, n_step, B, 5)
    ref = bref.branching_sampled(branching, ring, windows, n_step, 0.95, 1.0, double_q, [A])
    dqn = dqn_sampled(plain, ring, windows, n_step, 0.95, 1.0, double_q)
    np.testing.assert_allclose(ref["returns"], dqn["returns"], rtol=1e-14, atol=1e-14)
    np.testing.assert_allclose(ref["q"], dqn["q"], rtol=1e-14, atol=1e-14)
    for a, b in zip(ref["grads"], dqn["grads"]):
        np.testing.assert_allclose(a, b, rtol=1e-14, atol=1e-14)


# ------------------------------------------------------------------------ the model
def _env(action_space, observation_space=None):
    env = _Env(4, 1)
    env.env.action_space = {0: action_space}
    if observation_space is not None:
        env.env.observation_space = {0: observation_space}
    return env


def _make(env, **cfg):
    from warp_drive_b200.training.models.fully_connected import ModelFactory

    cfg = {"type": "fully_connected_branching_q", "fc_dims": [8], **cfg}
    return ModelFactory.create(cfg["type"])(env=env, model_config=cfg, policy="shared",
                                            policy_tag_to_agent_id_map={"shared": [0]})


def test_model_shapes_and_checkpoints_load_across_types():
    from warp_drive_b200.utils import spaces as sp

    m = _make(_env(sp.MultiDiscrete([5, 3])))
    assert m.is_q_network and m.branch_sizes == [5, 3] and m.policy_head.out_features == 8
    assert [n for n, _ in m.named_parameters()] == [
        "fc.0.0.weight", "fc.0.0.bias", "policy_head.weight", "policy_head.bias"]
    x = torch.randn(6, 4)
    (q,), v = m(x)
    assert v is None and q.shape == (6, 8)
    assert [t.shape[-1] for t in m.branches(q)] == [5, 3]
    # D = 1: FullyConnectedQ's weights at the same seed, and checkpoints in both directions
    torch.manual_seed(11)
    one = _make(_env(sp.Discrete(4)))
    torch.manual_seed(11)
    plain = _make(_env(sp.Discrete(4)), type="fully_connected_q")
    for a, b in zip(one.state_dict().values(), plain.state_dict().values()):
        assert torch.equal(a, b)
    torch.manual_seed(12)
    other = _make(_env(sp.Discrete(4)), type="fully_connected_q")
    one.load_state_dict(other.state_dict())
    plain.load_state_dict(one.state_dict())
    assert torch.equal(plain(x)[0][0], other(x)[0][0])


@pytest.mark.parametrize("key,value", [
    ("dueling", True), ("stream_fc_dims", [8]), ("noisy", True), ("noisy_sigma0", 0.4),
    ("masked", True), ("num_quantiles", 8), ("num_cosines", 8), ("num_tau_samples", 8),
    ("num_tau_prime_samples", 8), ("num_quantile_samples", 8), ("num_atoms", 51),
    ("v_min", -10.0), ("v_max", 10.0)])
def test_model_refuses_the_other_q_heads_keys(key, value):
    from warp_drive_b200.utils import spaces as sp

    with pytest.raises(ValueError, match=f"model.{key}"):
        _make(_env(sp.MultiDiscrete([5, 3])), **{key: value})


def test_model_refuses_box_actions_and_action_masks():
    from warp_drive_b200.utils import spaces as sp

    with pytest.raises(ValueError, match="Discrete or MultiDiscrete"):
        _make(_env(sp.Box(-1.0, 1.0, shape=(2,), dtype=np.float32)))
    masked = sp.Dict({"obs": sp.Box(-1.0, 1.0, shape=(4,), dtype=np.float32),
                      "action_mask": sp.Box(0.0, 1.0, shape=(8,), dtype=np.float32)})
    with pytest.raises(ValueError, match="action_mask"):
        _make(_env(sp.MultiDiscrete([5, 3]), masked))


def test_pass_selection_and_one_launch_rollout_eligibility():
    _lib_or_skip()
    from warp_drive_b200.training.algorithms import fused_dqn as fd
    from warp_drive_b200.training.algorithms.dqn import BranchingDQN
    from warp_drive_b200.training.fused_single_agent import FusedSingleAgentRollout
    from warp_drive_b200.utils import spaces as sp

    algo = BranchingDQN(0.99, n_step=3)
    multi = _make(_env(sp.MultiDiscrete([5, 3])))
    one = _make(_env(sp.Discrete(2)))
    for q in (multi, one):
        assert fd.FusedBranchingDQNUpdate.supported(algo, q, 8, 2, 100, 256)
        assert not fd.FusedDQNUpdate.supported(algo, q, 8, 2, 100, 256)
    assert fd._shape_struct(algo, multi, 8, 2, 100).n_actions == 8
    # outside the envelope: the torch loss
    assert not fd.FusedBranchingDQNUpdate.supported(
        algo, _make(_env(sp.MultiDiscrete([40, 25]))), 8, 2, 100, 256)
    assert not fd.FusedBranchingDQNUpdate.supported(
        algo, _make(_env(sp.MultiDiscrete([2] * 17))), 8, 2, 100, 256)

    class _W:
        n_agents = 1

        class env:
            name = "ClassicControlCartPoleEnv"

    assert FusedSingleAgentRollout.eligible(_W, {"shared": one}, {"shared": [0]})
    assert not FusedSingleAgentRollout.eligible(_W, {"shared": multi}, {"shared": [0]})


def test_run_config_loads():
    from warp_drive_b200.training.trainer import load_run_config

    cfg = load_run_config("tag_continuous_dqn")
    base = load_run_config("tag_continuous")
    env = dict(base["env"], num_other_agents_observed=8)
    assert cfg["env"] == env
    assert set(cfg["policy"]) == {"runner", "tagger"}
    for pol in cfg["policy"].values():
        assert pol["algorithm"] == "DQN"
        assert pol["model"]["type"] == "fully_connected_branching_q"
        assert pol["model"]["fc_dims"] == [64, 64]
    assert cfg["trainer"]["replay_slots_per_env"] > 0
    assert "epsilon" in cfg["sampler"]["params"]
    # F = 7 K + 1 for K observed agents: the native envelope's F <= 63
    assert 7 * env["num_other_agents_observed"] + 1 <= 63


# ------------------------------------------------------------------------ ABI
def test_struct_layout_and_bindings_match_the_header(tmp_path):
    from warp_drive_b200 import lib as wlib

    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "wdb200.h"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(wdb_q_branches));',
             '  printf("n_heads %zu\\n", offsetof(wdb_q_branches, n_heads));',
             '  printf("sizes %zu\\n", offsetof(wdb_q_branches, sizes));',
             '  printf("count %zu\\n", sizeof(((wdb_q_branches *)0)->sizes) / sizeof(int));',
             "  return 0;", "}"]
    (tmp_path / "layout.c").write_text("\n".join(lines))
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(tmp_path / "layout"),
                    str(tmp_path / "layout.c")], check=True)
    out = subprocess.run([str(tmp_path / "layout")], check=True, capture_output=True,
                         text=True).stdout
    got = {k: int(v) for k, v in (line.split() for line in out.splitlines())}
    assert ctypes.sizeof(wlib.QBranches) == got["size"]
    assert [n for n, _ in wlib.QBranches._fields_] == ["n_heads", "sizes"]
    assert wlib.QBranches.n_heads.offset == got["n_heads"]
    assert wlib.QBranches.sizes.offset == got["sizes"]
    assert wlib.Q_MAX_BRANCHES == got["count"]

    squash = re.sub(r"\s+", " ", header)
    want = [
        "int wdb_sample_epsilon_greedy_branching(void *stream, void *rng_state, const float "
        "*q_values, const wdb_q_branches *branches, int *actions, long long n_rows, float "
        "epsilon, const unsigned int *words);",
        "int wdb_branching_dqn_update_sampled_supported(const wdb_dqn_update_args *update, const "
        "wdb_q_branches *branches, int n_windows);",
        "long long wdb_branching_dqn_update_sampled_workspace_bytes(const wdb_dqn_update_args "
        "*update, const wdb_q_branches *branches, int n_windows);",
        "int wdb_branching_dqn_update_sampled(void *stream, const wdb_dqn_update_args *update, "
        "const wdb_q_branches *branches, const wdb_replay_windows *windows);",
        "int wdb_branching_dqn_update_prioritized_supported(const wdb_dqn_update_args *update, "
        "const wdb_q_branches *branches, int n_windows);",
        "long long wdb_branching_dqn_update_prioritized_workspace_bytes(const wdb_dqn_update_args "
        "*update, const wdb_q_branches *branches, int n_windows);",
        "int wdb_branching_dqn_update_prioritized(void *stream, const wdb_dqn_update_args "
        "*update, const wdb_q_branches *branches, const wdb_replay_windows *windows, const float "
        "*weights);",
    ]
    for proto in want:
        assert proto in squash, proto
    sig = wlib._SIGNATURES
    i, ll, f, vp = ctypes.c_int, ctypes.c_longlong, ctypes.c_float, ctypes.c_void_p
    u, b = ctypes.POINTER(wlib.DqnUpdate), ctypes.POINTER(wlib.QBranches)
    w = ctypes.POINTER(wlib.ReplayWindows)
    assert sig["wdb_sample_epsilon_greedy_branching"] == (i, [vp, vp, vp, b, vp, ll, f, vp])
    for kind in ("sampled", "prioritized"):
        assert sig[f"wdb_branching_dqn_update_{kind}_supported"] == (i, [u, b, i])
        assert sig[f"wdb_branching_dqn_update_{kind}_workspace_bytes"] == (ll, [u, b, i])
    assert sig["wdb_branching_dqn_update_sampled"] == (i, [vp, u, b, w])
    assert sig["wdb_branching_dqn_update_prioritized"] == (i, [vp, u, b, w, vp])


def _shape(sizes, F=57, dims=(64, 64)):
    from warp_drive_b200 import lib as wlib

    u = wlib.DqnUpdate()
    u.n_envs, u.n_agents, u.obs_dim, u.n_actions = 64, 2, F, int(sum(sizes))
    u.capacity, u.n_step, u.gamma, u.huber_delta, u.double_q = 100, 3, 0.99, 1.0, 1
    for net in (u.q, u.target_q):
        net.n_hidden = len(dims)
        for k, width in enumerate(dims):
            net.widths[k] = width
    b = wlib.QBranches()
    b.n_heads = len(sizes)                  # more than 16: the struct holds the first 16
    for d, a in enumerate(sizes[:wlib.Q_MAX_BRANCHES]):
        b.sizes[d] = a
    return u, b


def test_supported_at_the_envelopes_edges():
    wlib = _lib_or_skip()
    L = wlib.load()

    def ok(sizes, B=256, **kw):
        u, b = _shape(sizes, **kw)
        got = L.wdb_branching_dqn_update_sampled_supported(ctypes.byref(u), ctypes.byref(b), B)
        assert got == L.wdb_branching_dqn_update_prioritized_supported(
            ctypes.byref(u), ctypes.byref(b), B)
        nbytes = L.wdb_branching_dqn_update_sampled_workspace_bytes(
            ctypes.byref(u), ctypes.byref(b), B)
        assert (nbytes > 0) == bool(got)
        if len(sizes) <= 16:               # valid branches: DQN's envelope and workspace
            assert got == L.wdb_dqn_update_sampled_supported(ctypes.byref(u), B)
            assert nbytes == L.wdb_dqn_update_sampled_workspace_bytes(ctypes.byref(u), B)
        return bool(got)

    assert ok([21, 21]) and ok([5, 3]) and ok([64]) and ok([1])
    assert ok([32, 32]) and not ok([32, 33])                          # A 64 / 65
    assert ok([4] * 16) and not ok([2] * 17)                          # D 16 / 17
    assert ok([21, 21], F=63) and not ok([21, 21], F=64)              # F 63 / 64
    assert ok([21, 21], dims=()) and ok([21, 21], dims=(32, 32, 32))
    assert not ok([21, 21], dims=(64, 64, 64))        # DQN's shared-memory limit at F = 57
    assert not ok([21, 21], dims=(65,)) and not ok([21, 21], B=0)
    assert ok([21, 21], B=50000)
    for bad in ([5, 0, 3], [0], [5, -1]):                            # a head of size 0
        u, b = _shape(bad)
        u.n_actions = 8
        assert L.wdb_branching_dqn_update_sampled_supported(
            ctypes.byref(u), ctypes.byref(b), 256) == 0
    u, b = _shape([5, 3])
    b.n_heads = 0
    assert L.wdb_branching_dqn_update_sampled_supported(ctypes.byref(u), ctypes.byref(b), 256) == 0
    u, b = _shape([5, 3])
    u.n_actions = 9                                                   # sum A_d != A
    assert L.wdb_branching_dqn_update_sampled_supported(ctypes.byref(u), ctypes.byref(b), 256) == 0
    # no launch without weights, windows or valid branches; none with a bad epsilon
    u, b = _shape([5, 3])
    w = wlib.ReplayWindows()
    w.n_windows = 8
    assert L.wdb_branching_dqn_update_prioritized(None, u, b, ctypes.byref(w), None) == 1
    assert L.wdb_branching_dqn_update_sampled(None, u, b, None) == 1
    assert L.wdb_branching_dqn_update_sampled(None, u, None, ctypes.byref(w)) == 1
    assert L.wdb_sample_epsilon_greedy_branching(None, None, None, b, None, 4, 0.5, None) == 1
    assert L.wdb_sample_epsilon_greedy_branching(None, None, None, None, None, 4, 0.5, None) == 1


# ------------------------------------------------------------------------ ptxas
# Registers under nvcc 12.9 at sm_90a (-O3): branching_q_pass_kernel and
# branching_q_prioritized_kernel 130 each, epsilon_greedy_branching_kernel 34,
# ddpg_reduce_kernel 32.
_KERNELS = ("epsilon_greedy_branching_kernel", "branching_q_pass_kernel",
            "branching_q_prioritized_kernel", "ddpg_reduce_kernel")


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_kernels_compile_for_sm90a_without_spills(tmp_path):
    out = str(tmp_path / "branching_q.cubin")
    proc = subprocess.run(NVCC_SM90A + ["-Xptxas", "-v", "-cubin", "-I",
                                        os.path.join(ROOT, "include"),
                                        os.path.join(CSRC, "wdb_branching_q.cu"), "-o", out],
                          capture_output=True, text=True, check=True)
    stats, name = {}, None
    for line in proc.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            stats[name] = (int(m.group(1)), int(m.group(2)))
    assert len(stats) == len(_KERNELS), stats
    for k in _KERNELS:
        hits = [v for n, v in stats.items() if k in n]
        assert hits == [(0, 0)], (k, stats)
    # the tests that find DQN's kernels by name must not find these
    assert not any("dqn_pass_kernel" in n or "dqn_weighted_kernel" in n for n in stats)
