"""Prioritized replay's host side without a GPU: the float64 reference (tests/per_reference.py)
-- its descent against a brute-force prefix search, its admit ranges against the definition of
a valid window, the weighted DQN update against torch autograd through the real DQN and
FullyConnectedQ -- the trainer keys' validation and refusals, the new ABI struct, the entry
points' argument refusals, and the new kernels' resource use."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import dqn_update_reference as dqn_ref
import per_reference as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "warp_drive_b200", "csrc")


def _leaves(n, seed, zero_share=0.5, decades=12):
    g = np.random.default_rng(seed)
    p = (10.0 ** g.uniform(-decades / 2, decades / 2, n)).astype(np.float32)
    p[g.random(n) < zero_share] = 0
    return p


@pytest.mark.parametrize("n", [1, 31, 32, 33, 1000, 32 ** 2 + 5, 40000])
def test_tree_levels_are_pairwise_sums_of_the_children(n):
    leaves = _leaves(n, n)
    levels = ref.build_tree(leaves)
    assert len(levels[-1]) == 1 and len(levels) == ref.n_levels(n)
    below = leaves.astype(np.float64)
    for lv in levels:
        assert len(lv) == -(-len(below) // 32)
        for j in (0, len(lv) - 1):
            kids = np.zeros(32)
            part = below[32 * j:32 * j + 32]
            kids[:len(part)] = part
            h = 16
            while h >= 1:                                  # the warp's shuffle-down order
                kids[:h] = kids[:h] + kids[h:2 * h]
                h //= 2
            assert lv[j] == kids[0]
        below = lv
    assert levels[-1][0] == pytest.approx(leaves.astype(np.float64).sum(), rel=1e-12)


@pytest.mark.parametrize("n,zero_share", [(1000, 0.5), (40000, 0.9), (5000, 0.0)])
def test_descent_agrees_with_a_brute_force_prefix_search(n, zero_share):
    leaves = _leaves(n, 7 + n, zero_share)
    levels = ref.build_tree(leaves)
    S = levels[-1][0]
    g = np.random.default_rng(n)
    u = np.sort(g.uniform(0, S, 20000))
    ends = np.cumsum(leaves.astype(np.float64))
    # points a rounding of the two summation orders cannot move across a leaf boundary
    gap = np.abs(ends[np.searchsorted(ends, u).clip(0, n - 1)] - u)
    gap = np.minimum(gap, np.abs(ends[(np.searchsorted(ends, u) - 1).clip(0, n - 1)] - u))
    clear = gap > 1e-9 * S
    assert clear.mean() > 0.99
    got = ref.descend(leaves, levels, u)
    want = ref.brute_force_leaf(leaves, u)
    assert (got[clear] == want[clear]).all()
    assert (leaves[got] > 0).all()                           # never a zero leaf
    # at and past the total: the last positive leaf
    last = np.flatnonzero(leaves > 0)[-1]
    assert (ref.descend(leaves, levels, np.array([S, S * (1 + 1e-12), 1e300])) == last).all()


def test_descent_never_returns_a_zero_leaf_around_a_single_positive_leaf():
    for n in (1, 32, 1025, 40000):
        for at in sorted({0, n // 2, n - 1}):
            leaves = np.zeros(n, dtype=np.float32)
            leaves[at] = 3e-30
            levels = ref.build_tree(leaves)
            u = np.array([0.0, levels[-1][0] * 0.5, levels[-1][0], 1.0])
            assert (ref.descend(leaves, levels, u) == at).all(), (n, at)


def test_stratified_points_land_in_their_strata():
    B, S = 4096, 123.456
    u01 = ref.uniform53(ref.philox_words(11, 3, B))
    assert (u01 >= 0).all() and (u01 < 1).all()
    u, lo, hi = ref.segment_points(S, u01)
    assert (u >= lo).all() and (u <= hi).all()
    assert np.all(np.diff(lo) > 0) and hi[-1] == S


@pytest.mark.parametrize("C,T,n_step,E", [(7, 4, 3, 3), (20, 4, 3, 2), (13, 1, 5, 2),
                                          (9, 8, 1, 1)])
def test_admit_marks_exactly_the_valid_windows(C, T, n_step, E):
    """A sequence of rollouts across the seam (C = T + n_step wraps on every rollout): after
    each admit, a leaf is positive exactly when its window is valid, and a leaf written by
    set_priorities keeps its value until its slot is rewritten."""
    leaves = np.zeros(C * E, dtype=np.float32)
    cursor, filled, p_max = 0, 0, np.float32(1.0)
    for r in range(3 * C):
        before = (cursor, filled)
        cursor, filled = (cursor + T) % C, min(C, filled + T)
        leaves = ref.admit(leaves, p_max, 0.6, C, E, n_step, before, (cursor, filled))
        oldest = cursor if filled == C else 0
        ok = np.repeat(ref.valid_starts(C, oldest, filled, n_step), E)
        assert ((leaves > 0) == ok).all(), (r, before, cursor, filled)
        if r == 2 and ok.any():              # a priority write, then later rollouts
            w = np.array([[s, 0] for s in np.flatnonzero(ok[::E])[:1]], dtype=np.int32)
            leaves, p_max = ref.set_priorities(leaves, p_max, w, [5.0], [1.0], 0.6, 1e-6, C,
                                               E, n_step, oldest, filled)
            assert p_max == np.float32(4.0 + 1e-6)


def test_set_priorities_keeps_the_largest_duplicate_and_skips_invalid_windows():
    C, E, n_step = 10, 2, 2
    leaves = np.full(C * E, 0.5, dtype=np.float32)
    w = np.array([[3, 1], [3, 1], [3, 1], [9, 0], [2, 0]], dtype=np.int32)
    q = np.array([1.0, 4.0, 2.0, 9.0, 0.0], dtype=np.float32)
    r = np.zeros(5, dtype=np.float32)
    # filled 10, oldest 0: starts 8 and 9 lack their look-ahead
    out, p_max = ref.set_priorities(leaves, np.float32(1.0), w, q, r, 1.0, 0.0, C, E, n_step, 0,
                                    10)
    assert out[3 * E + 1] == 4.0 and out[2 * E] == 0.0 and out[9 * E] == 0.5
    assert p_max == 4.0
    for perm in ([1, 0, 2, 3, 4], [2, 1, 0, 4, 3]):
        again, _ = ref.set_priorities(leaves, np.float32(1.0), w[perm], q[perm], r[perm], 1.0,
                                      0.0, C, E, n_step, 0, 10)
        assert (again == out).all()


def test_weights_are_normalised_by_the_batch_maximum():
    p = np.array([0.5, 2.0, 0.25, 1.0])
    w = ref.weights(p, 0.4)
    assert w.max() == 1.0 and w[2] == 1.0
    assert w[1] == pytest.approx((2.0 / 0.25) ** -0.4)
    assert (ref.weights(p, 0.0) == 1).all()


@pytest.mark.parametrize("double_q", [True, False], ids=["double_q", "max_target"])
@pytest.mark.parametrize("n_step,Np,dims", [(1, 1, [8, 8]), (3, 2, [6]), (2, 1, [])])
def test_weighted_reference_matches_torch_autograd(double_q, n_step, Np, dims):
    from warp_drive_b200.training.algorithms.dqn import DQN
    from test_dqn_cpu import _windows

    C, E, F, A, gamma = 13, 3, 4, 3, 0.93
    q_net, target = dqn_ref.make_q_models(F, A, dims, seed=n_step)
    with torch.no_grad():
        for p in target.parameters():
            p.add_(0.3 * torch.randn_like(p))
    ring = dqn_ref.make_q_ring(C, E, Np, F, A, seed=n_step)
    windows = _windows(C, E * Np, n_step)
    B = len(windows)
    w = np.random.default_rng(n_step).uniform(0.05, 1.0, B)
    probe = dqn_ref.dqn_sampled((q_net, target), ring, windows, n_step, gamma, 1e9, double_q)
    delta = float(np.median(np.abs(probe["diff"])))
    want = ref.dqn_weighted((q_net, target), ring, windows, w, n_step, gamma, delta, double_q)
    algo = DQN(gamma, n_step=n_step, double_q=double_q, huber_delta=delta)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x))  # noqa: E731
    obs, actions, rewards, done, boot_obs = dqn_ref.gather(ring, windows, n_step, Np)
    q_net.zero_grad()
    loss, _, _ = algo.loss(q_net, target, t(obs), t(actions)[:, None], t(rewards),
                           t(done).double(), t(boot_obs), weights=t(w))
    loss.backward()
    assert abs(loss.item() - want["sum_huber"] / B) <= 1e-12
    got = [p.grad.numpy() for p in q_net.parameters()]
    assert len(got) == len(want["grads"])
    for a, b in zip(got, want["grads"]):
        assert np.abs(a - b).max() <= 1e-12
    # unit weights: the unweighted loss and reference
    ones = ref.dqn_weighted((q_net, target), ring, windows, np.ones(B), n_step, gamma, delta,
                            double_q)
    plain = dqn_ref.dqn_sampled((q_net, target), ring, windows, n_step, gamma, delta, double_q)
    assert ones["sum_huber"] == plain["sum_huber"]
    for a, b in zip(ones["grads"], plain["grads"]):
        assert np.array_equal(a, b)
    l1, _, _ = algo.loss(q_net, target, t(obs), t(actions)[:, None], t(rewards),
                         t(done).double(), t(boot_obs), weights=torch.ones(B, dtype=torch.float64))
    l0, _, _ = algo.loss(q_net, target, t(obs), t(actions)[:, None], t(rewards),
                         t(done).double(), t(boot_obs))
    assert l1.item() == pytest.approx(l0.item(), rel=1e-15)


def test_prioritized_settings_validation():
    from warp_drive_b200.training.trainer_ddpg import prioritized_settings

    replay = {"slots": 100, "batch_rows": 64, "updates": 1, "warmup": 10}
    assert prioritized_settings({}, replay) is None
    assert prioritized_settings({"prioritized_replay": False}, None) is None
    got = prioritized_settings({"prioritized_replay": True}, replay)
    assert (got["alpha"], got["epsilon"]) == (0.6, 1e-6)
    assert got["beta"].get_param_value(10 ** 9) == 0.5
    got = prioritized_settings({"prioritized_replay": True, "priority_alpha": 0,
                                "priority_beta": [[0, 0.4], [100, 1.0]],
                                "priority_epsilon": 0.01}, replay)
    assert got["alpha"] == 0.0 and got["epsilon"] == 0.01
    assert got["beta"].get_param_value(50) == pytest.approx(0.7)
    on = {"prioritized_replay": True}
    for bad, replay_, match in (
            ({"priority_alpha": 0.5}, replay, "priority_alpha needs prioritized_replay"),
            ({"priority_beta": 0.5}, replay, "priority_beta needs prioritized_replay"),
            ({"priority_epsilon": 0.1}, replay, "priority_epsilon needs prioritized_replay"),
            (on, None, "needs replay_slots_per_env"),
            ({"prioritized_replay": "yes"}, replay, "True or False"),
            (dict(on, priority_alpha=1.5), replay, "priority_alpha"),
            (dict(on, priority_alpha=-0.1), replay, "priority_alpha"),
            (dict(on, priority_alpha=True), replay, "priority_alpha"),
            (dict(on, priority_beta=1.2), replay, "priority_beta"),
            (dict(on, priority_beta=[[0, 0.4], [10, 1.1]]), replay, "priority_beta"),
            (dict(on, priority_beta=[[10, 0.4], [0, 1.0]]), replay, "increasing"),
            (dict(on, priority_beta=[]), replay, "priority_beta"),
            (dict(on, priority_epsilon=0), replay, "priority_epsilon"),
            (dict(on, priority_epsilon=-1e-6), replay, "priority_epsilon"),
            (dict(on, priority_epsilon=float("inf")), replay, "priority_epsilon")):
        with pytest.raises(ValueError, match=match):
            prioritized_settings(bad, replay_)


@pytest.mark.parametrize("cls_name", ["TrainerDDPG", "TrainerTD3", "TrainerSAC"])
def test_actor_critic_trainers_refuse_prioritized_replay(cls_name):
    import importlib

    module = {"TrainerDDPG": "trainer_ddpg", "TrainerTD3": "trainer_td3",
              "TrainerSAC": "trainer_sac"}[cls_name]
    cls = getattr(importlib.import_module(f"warp_drive_b200.training.{module}"), cls_name)
    tr = object.__new__(cls)
    tr.training_batch_size_per_env = 8
    cfg = {"n_step": 3, "replay_slots_per_env": 100}
    assert tr._batch_slots_per_env(dict(cfg)) == 100 and tr.prioritized is None
    with pytest.raises(ValueError, match="prioritized_replay is DQN's"):
        tr._batch_slots_per_env(dict(cfg, prioritized_replay=True))


def test_dqn_trainer_takes_prioritized_replay():
    from warp_drive_b200.training.trainer_dqn import TrainerDQN

    tr = object.__new__(TrainerDQN)
    tr.training_batch_size_per_env = 8
    assert tr._batch_slots_per_env({"n_step": 3, "replay_slots_per_env": 100,
                                    "prioritized_replay": True}) == 100
    assert tr.prioritized["alpha"] == 0.6
    with pytest.raises(ValueError, match="needs replay_slots_per_env"):
        tr._batch_slots_per_env({"n_step": 3, "prioritized_replay": True})


def test_prioritized_run_config_loads():
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_ddpg import prioritized_settings, replay_settings

    cfg = load_run_config("single_cartpole_dqn_prioritized")
    base = load_run_config("single_cartpole_dqn")
    t = cfg["trainer"]
    extra = {k: v for k, v in t.items() if k not in base["trainer"]}
    assert set(extra) == {"prioritized_replay", "priority_alpha", "priority_beta",
                          "priority_epsilon"}
    assert {k: v for k, v in t.items() if k in base["trainer"]} == base["trainer"]
    assert cfg["policy"] == base["policy"] and cfg["sampler"] == base["sampler"]
    got = prioritized_settings(t, replay_settings(t, t["train_batch_size"] // t["num_envs"],
                                                  t["n_step"]))
    assert got["beta"].get_param_value(0) == 0.4 and got["beta"].get_param_value(10 ** 9) == 1.0
    assert got["alpha"] == 0.6 and got["epsilon"] == 1e-6


def test_per_store_struct_layout(tmp_path):
    from warp_drive_b200 import lib as wlib
    from test_abi_layout_cpu import _c_fields

    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    fields = _c_fields(header, "wdb_per_store")
    assert [n for n, _ in wlib.PerStore._fields_] == fields
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "wdb200.h"',
             "int main(void) {", '  printf("size %zu\\n", sizeof(wdb_per_store));']
    lines += [f'  printf("{f} %zu\\n", offsetof(wdb_per_store, {f}));' for f in fields]
    lines += ["  return 0;", "}"]
    (tmp_path / "layout.c").write_text("\n".join(lines))
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(tmp_path / "layout"),
                    str(tmp_path / "layout.c")], check=True)
    out = subprocess.run([str(tmp_path / "layout")], check=True, capture_output=True,
                         text=True).stdout
    got = dict((k, int(v)) for k, v in (line.split() for line in out.splitlines()))
    assert ctypes.sizeof(wlib.PerStore) == got["size"]
    for f in fields:
        assert getattr(wlib.PerStore, f).offset == got[f], f


def _lib_or_skip():
    from warp_drive_b200 import lib as wlib

    if not os.path.exists(wlib.LIB_PATH):
        pytest.skip("libwdb200.so is not built")
    return wlib, wlib.load()


def test_tree_sizes_and_argument_refusals():
    """Every refusal returns cudaErrorInvalidValue (1) before any CUDA call, so it runs here."""
    wlib, L = _lib_or_skip()
    for n in (1, 31, 32, 33, 1025, 40000, 10 ** 6, 2 ** 31 - 1):
        count, nodes, lv = n, 0, 0
        while True:
            count = -(-count // 32)
            nodes, lv = nodes + count, lv + 1
            if count == 1:
                break
        assert L.wdb_per_nodes(n) == nodes and L.wdb_per_levels(n) == lv, n
        if n <= 40000:
            assert lv == ref.n_levels(n) and nodes == len(ref.flat_nodes(
                ref.build_tree(np.zeros(n, np.float32))))
    for n in (0, -1, 2 ** 31):
        assert L.wdb_per_nodes(n) == -1 and L.wdb_per_levels(n) == -1

    fake = 1 << 40                                      # never dereferenced: refused first

    def store(**kw):
        s = wlib.PerStore()
        s.capacity, s.n_rows, s.n_step, s.alpha, s.epsilon = 10, 4, 3, 0.6, 1e-6
        s.leaves = s.nodes = s.p_max = fake
        for k, v in kw.items():
            setattr(s, k, v)
        return ctypes.byref(s)

    bad_stores = [store(capacity=2 ** 20, n_rows=2 ** 11), store(capacity=3), store(n_rows=0),
                  store(n_step=0), store(alpha=1.5), store(alpha=-0.1),
                  store(alpha=float("nan")), store(epsilon=0.0), store(leaves=None),
                  store(nodes=None), store(p_max=None)]
    for s in bad_stores:
        assert L.wdb_per_admit(None, s, 0, 0, 4, 4) == 1
        assert L.wdb_per_sample_windows(None, s, fake, fake, fake, 8, 1, 1, fake) == 1
        assert L.wdb_per_set_priorities(None, s, fake, 8, fake, fake, 0, 8) == 1
    ok = store()
    for args in ((0, 0, 0, 0), (0, 0, 8, 8), (0, 0, 4, 5), (-1, 0, 4, 4), (0, 0, 10, 10),
                 (2, 2, 6, 5), (0, 11, 4, 10), (3, 0, 7, 4)):
        assert L.wdb_per_admit(None, ok, *args) == 1, args     # T < 1, T + n_step > C, ...
    for p in ((None, fake, fake, 8, fake), (fake, None, fake, 8, fake),
              (fake, fake, None, 8, fake), (fake, fake, fake, 0, fake),
              (fake, fake, fake, 8, None)):
        assert L.wdb_per_sample_windows(None, ok, p[0], p[1], p[2], p[3], 1, 1, p[4]) == 1
    for args in ((None, 8, fake, fake, 0, 8), (fake, 0, fake, fake, 0, 8),
                 (fake, 8, None, fake, 0, 8), (fake, 8, fake, None, 0, 8),
                 (fake, 8, fake, fake, 10, 8), (fake, 8, fake, fake, -1, 8),
                 (fake, 8, fake, fake, 0, 11), (fake, 8, fake, fake, 0, 3)):
        assert L.wdb_per_set_priorities(None, ok, *args) == 1, args


def test_prioritized_pass_takes_the_sampled_shapes():
    wlib, L = _lib_or_skip()
    from warp_drive_b200.training.algorithms.dqn import DQN
    from warp_drive_b200.training.algorithms.fused_dqn import _shape_struct

    for dims, F, A, C, n_step, B in (((64, 64), 4, 2, 100, 3, 512), ((), 4, 2, 100, 3, 16),
                                     ((65,), 4, 2, 100, 3, 8), ((8,), 64, 2, 100, 3, 8),
                                     ((8,), 4, 2, 3, 3, 8), ((8,), 4, 2, 100, 3, 0)):
        q, _ = dqn_ref.make_q_models(F, A, list(dims))
        u = ctypes.byref(_shape_struct(DQN(0.99, n_step=n_step), q, 8, 1, C))
        assert (L.wdb_dqn_update_prioritized_supported(u, B)
                == L.wdb_dqn_update_sampled_supported(u, B))
        assert (L.wdb_dqn_update_prioritized_workspace_bytes(u, B)
                == L.wdb_dqn_update_sampled_workspace_bytes(u, B))
    q, _ = dqn_ref.make_q_models(4, 2, [8])
    u = ctypes.byref(_shape_struct(DQN(0.99, n_step=3), q, 8, 1, 100))
    w = wlib.ReplayWindows()
    w.n_windows = 8
    assert L.wdb_dqn_update_prioritized(None, u, ctypes.byref(w), None) == 1   # no weights


PINNED = ("dqn_pass_kernel", "replay_sample_windows_kernel", "ddpg_reduce_kernel",
          "epsilon_greedy_kernel", "ddpg_update_kernel", "td3_critic_kernel", "td3_actor_kernel",
          "sac_critic_kernel", "sac_actor_kernel")


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_new_kernels_compile_without_spills_and_have_names_of_their_own(tmp_path):
    flags = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
             "-Xptxas", "-v", "-cubin"]
    want = {"wdb_ddpg_update.cu": ["dqn_weighted_kernel"],
            "wdb_per.cu": ["per_repair_kernel", "per_admit_kernel", "per_sample_kernel",
                           "per_weights_kernel", "per_clear_kernel", "per_write_kernel"]}
    for src, kernels in want.items():
        err = subprocess.run(flags + [os.path.join(CSRC, src), "-o", str(tmp_path / "k.cubin")],
                             capture_output=True, text=True, check=True).stderr
        blocks = re.split(r"Compiling entry function '", err)[1:]
        for k in kernels:
            hits = [b for b in blocks if k in b.split("'")[0]]
            assert len(hits) == 1, (k, src)
            assert "0 bytes spill stores, 0 bytes spill loads" in hits[0], (k, hits[0])
            assert not any(p in hits[0].split("'")[0] for p in PINNED), k
