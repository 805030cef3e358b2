"""The replay buffer's host side without a GPU: the float64 reference of the sampled passes
(tests/replay_update_reference.py) against torch, the sampled n-step return against the ring's
regular windows, the trainer keys' validation, the new ABI struct and the new kernels' resource
use."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from replay_update_reference import ddpg_sampled, gather, sampled_returns
from test_ddpg_update_reference_cpu import make_models, make_ring

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "warp_drive_b200", "csrc")


def _windows(C, EN, n_step):
    """Every start slot (so windows wrap the physical end and a done flag set in one slot sits
    at each position of some window), two agent rows, and duplicates."""
    w = [(s, (3 * s + k) % EN) for s in range(C) for k in range(2)]
    return np.array(w + w[:5], dtype=np.int32)


@pytest.mark.parametrize("n_step,Np", [(1, 1), (3, 2), (5, 1)])
def test_reference_matches_torch_on_the_gathered_batch(n_step, Np):
    from warp_drive_b200.training.algorithms.ddpg import DDPG

    C, E, F, A, gamma = 11, 4, 3, 2, 0.9
    ring = make_ring(C, E, Np, F, A, done_slots=(4,), seed=n_step)
    windows = _windows(C, E * Np, n_step)
    obs, actions, rewards, done, boot_obs = gather(ring, windows, n_step, Np)
    B = len(windows)
    assert obs.shape == (B, F) and rewards.shape == (n_step, B) and boot_obs.shape == (B, F)
    # the gather, restated slot by slot
    for g, (s, n) in enumerate(windows):
        e, a = divmod(int(n), Np)
        assert (obs[g] == ring[0][s, e, a]).all() and (actions[g] == ring[1][s, e, a]).all()
        assert (boot_obs[g] == ring[0][(s + n_step) % C, e, a]).all()
        for j in range(n_step):
            assert rewards[j, g] == ring[2][(s + j) % C, e, a]
            assert done[j, g] == ring[3][(s + j) % C, e]
    assert done.any(axis=1).all()                      # a done flag at every position
    boot = np.random.default_rng(0).standard_normal(B)
    want = sampled_returns(rewards, done, boot, gamma)
    got = DDPG(gamma, n_step=n_step).sampled_returns(
        torch.from_numpy(rewards), torch.from_numpy(done), torch.from_numpy(boot))
    assert np.abs(got.numpy() - want).max() <= 1e-12
    # the whole DDPG update on the project's networks: duplicates count once per appearance
    models = make_models(F, A, [8, 8], [8, 8], seed=1)
    ref = ddpg_sampled(models, ring, windows, n_step, gamma)
    again = ddpg_sampled(models, ring, np.concatenate([windows, windows]), n_step, gamma)
    for a, b in zip(ref["critic_grads"] + ref["actor_grads"],
                    again["critic_grads"] + again["actor_grads"]):
        assert np.abs(a - b).max() <= 1e-12            # means: doubling the batch changes nothing
    assert again["sum_j"] == pytest.approx(2 * ref["sum_j"], rel=1e-12)


def test_sampled_return_is_the_rings_regular_window():
    from warp_drive_b200.training.algorithms.ddpg import DDPG

    T, E, n, gamma = 9, 5, 4, 0.97
    g = torch.Generator().manual_seed(0)
    rewards = torch.randn(T, E, 1, generator=g, dtype=torch.float64)
    done = (torch.rand(T, E, generator=g) < 0.3).to(torch.int32)
    boot = torch.randn(T - n + 1, E, 1, generator=g, dtype=torch.float64)
    algo = DDPG(gamma, n_step=n)
    ring = algo.window_returns(rewards, done, boot[:-1], boot[-1])
    for i in range(T - n):                              # every window but the last
        got = algo.sampled_returns(rewards[i:i + n, :, 0], done[i:i + n].double(), boot[i, :, 0])
        assert torch.equal(got, ring[i, :, 0])


def test_replay_settings_validation():
    from warp_drive_b200.training.trainer_ddpg import replay_settings

    assert replay_settings({"n_step": 5}, 8, 5) is None
    got = replay_settings({"replay_slots_per_env": 1000}, 8, 5)
    assert got == {"slots": 1000, "batch_rows": None, "updates": 1, "warmup": 13}
    got = replay_settings({"replay_slots_per_env": 13, "replay_batch_rows": 256,
                           "updates_per_iteration": 4, "replay_warmup_slots": 6}, 8, 5)
    assert got == {"slots": 13, "batch_rows": 256, "updates": 4, "warmup": 6}
    for bad, key in (({"replay_slots_per_env": 12}, "replay_slots_per_env"),
                     ({"replay_batch_rows": 4}, "replay_batch_rows"),
                     ({"updates_per_iteration": 2}, "updates_per_iteration"),
                     ({"replay_warmup_slots": 20}, "replay_warmup_slots"),
                     ({"replay_slots_per_env": 100, "replay_batch_rows": 0}, "replay_batch_rows"),
                     ({"replay_slots_per_env": 100, "replay_batch_rows": 2 ** 31},
                      "replay_batch_rows"),
                     ({"replay_slots_per_env": 100, "updates_per_iteration": 0},
                      "updates_per_iteration"),
                     ({"replay_slots_per_env": 100, "replay_warmup_slots": 5},
                      "replay_warmup_slots"),
                     ({"replay_slots_per_env": 100, "replay_warmup_slots": 101},
                      "replay_warmup_slots")):
        with pytest.raises(ValueError, match=key):
            replay_settings(bad, 8, 5)


@pytest.mark.parametrize("name", ["ddpg", "td3", "sac"])
def test_replay_run_configs_load(name):
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_ddpg import replay_settings

    cfg = load_run_config(f"single_pendulum_{name}_replay")
    t = cfg["trainer"]
    assert cfg["policy"]["shared"]["algorithm"] == name.upper()
    got = replay_settings(t, t["train_batch_size"] // t["num_envs"], t["n_step"])
    assert got["slots"] * t["num_envs"] >= 10 ** 6 and 256 <= got["batch_rows"] <= 4096
    assert got["updates"] > 1
    if name == "sac":
        assert cfg["policy"]["shared"]["lr"]["actor"] == 3e-4


def test_replay_windows_struct_layout():
    from warp_drive_b200 import lib as wlib

    assert ctypes.sizeof(wlib.ReplayWindows) == 16
    assert (wlib.ReplayWindows.windows.offset, wlib.ReplayWindows.n_windows.offset) == (0, 8)
    src = open(os.path.join(ROOT, "include", "wdb200.h")).read()
    m = re.search(r"typedef struct wdb_replay_windows \{(.*?)\} wdb_replay_windows;", src, re.S)
    assert re.findall(r"(\w+);", m.group(1)) == ["windows", "n_windows"]


def _td3_struct(B=None, **kw):
    from test_td3_cpu import _struct

    return _struct(**kw)


def test_sampled_supported_takes_the_ring_shapes_and_checks_the_windows():
    from warp_drive_b200 import lib as wlib

    if not os.path.exists(wlib.LIB_PATH):
        pytest.skip("libwdb200.so is not built")
    L = wlib.load()
    u = _td3_struct(C=1000, cursor=5000)                 # the cursor is not read
    for name in ("td3_critic_update", "td3_actor_update"):
        sup = getattr(L, f"wdb_{name}_sampled_supported")
        nbytes = getattr(L, f"wdb_{name}_sampled_workspace_bytes")
        assert sup(ctypes.byref(u), 1) == 1 and sup(ctypes.byref(u), 4096) == 1
        assert sup(ctypes.byref(u), 0) == 0 and nbytes(ctypes.byref(u), 0) == -1
        assert 0 < nbytes(ctypes.byref(u), 16) < nbytes(ctypes.byref(u), 4096)
        assert sup(ctypes.byref(_td3_struct(C=5, n_step=5)), 8) == 0      # needs n_step + 1 slots
        assert sup(ctypes.byref(_td3_struct(C=6, n_step=5)), 8) == 1
        assert sup(ctypes.byref(_td3_struct(ad=(65, 64), C=100)), 8) == 0
    assert L.wdb_td3_critic_update_supported(ctypes.byref(u)) == 0        # the ring pass reads it


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_sampled_pass_instantiations_compile_without_spills(tmp_path):
    flags = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
             "-Xptxas", "-v", "-cubin"]
    from test_td3_cpu import SAMPLED

    want = {"wdb_ddpg_update.cu": [k + SAMPLED for k in ("ddpg_update_kernel", "td3_critic_kernel",
                                                         "td3_actor_kernel", "sac_critic_kernel",
                                                         "sac_actor_kernel")],
            "wdb_core.cu": ["replay_sample_windows_kernel"]}
    for src, kernels in want.items():
        err = subprocess.run(flags + [os.path.join(CSRC, src), "-o", str(tmp_path / "k.cubin")],
                             capture_output=True, text=True, check=True).stderr
        blocks = re.split(r"Compiling entry function '", err)[1:]
        for k in kernels:
            hits = [b for b in blocks if k in b.split("'")[0]]
            assert len(hits) == 1, (k, src)
            assert "0 bytes spill stores, 0 bytes spill loads" in hits[0], (k, hits[0])
