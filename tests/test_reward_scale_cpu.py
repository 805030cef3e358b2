"""CPU tests of running reward scaling: the float32 scan reference against an independent
float64 torch expression, the policy keys and their refusals (every replay trainer included),
every existing run config without the keys, the buffers, the C interface and its ctypes mirror,
and what ptxas makes of the scan kernel (no spills, no contracted FMA)."""
import ctypes
import glob
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from reward_scale_reference import RunningReturns, scale_f32, scan_f32  # noqa: E402

CONFIGS = os.path.join(ROOT, "warp_drive_b200", "training", "run_configs")


def _episode_data(T, E, Np, seed):
    rng = np.random.default_rng(seed)
    rewards = (rng.normal(size=(T, E, Np)) * 5 - 3).astype(np.float32)
    done = (rng.uniform(size=(T, E)) < 0.2).astype(np.int32)
    done[rng.uniform(size=(T, E)) < 0.05] = 2          # MountainCar's goal flag
    carry = rng.normal(size=(E, Np)).astype(np.float32) * 20
    return rewards, done, carry


# ------------------------------------------------------------------------ the reference
@pytest.mark.parametrize("T,E,Np", [(1, 5, 1), (7, 33, 3), (250, 17, 2)])
def test_scan_reference_matches_a_float64_torch_expression(T, E, Np):
    import torch

    rewards, done, carry = _episode_data(T, E, Np, seed=T + E + Np)
    gamma = 0.95
    got, carry_out = scan_f32(rewards, done, gamma, carry)
    assert got.dtype == np.float32 and carry_out.dtype == np.float32
    r, d = torch.tensor(rewards, dtype=torch.float64), torch.tensor(done) > 0
    c = torch.tensor(carry, dtype=torch.float64)
    want = torch.empty_like(r)
    for t in range(T):
        want[t] = gamma * c + r[t]
        c = torch.where(d[t][:, None], torch.zeros_like(c), want[t])
    bound = 1e-5 * (np.abs(rewards).max() / (1 - gamma) + np.abs(carry).max())
    assert np.abs(got - want.numpy()).max() <= bound
    assert np.abs(carry_out - c.numpy()).max() <= bound
    # a done step restarts the next step's return from its own reward: accumulate, record,
    # then zero
    t, e = np.nonzero(done[:-1] > 0)[0][:1], np.nonzero(done[:-1] > 0)[1][:1]
    if len(t):
        assert np.array_equal(got[t[0] + 1, e[0]], rewards[t[0] + 1, e[0]])


def test_scan_reference_rounds_the_multiply_and_the_add_apart():
    # 1 + 2^-23 squared needs more than 24 bits: a fused multiply-add keeps the low bit the
    # separate multiply rounds away
    g = np.float32(1 + 2.0 ** -23)
    c = np.full((1, 1), g, np.float32)
    r = np.full((1, 1, 1), -1.0, np.float32)
    got, _ = scan_f32(r, np.zeros((1, 1), np.int32), g, c)
    assert got[0, 0, 0] == np.float32(2.0 ** -22)
    assert float(g) * float(g) - 1.0 != float(got[0, 0, 0])       # the fused result


def test_running_returns_statistics_and_scale():
    E, Np, clip = 9, 2, 3.0
    run = RunningReturns(E, Np, 0.9, clip)
    all_returns = []
    for k in range(3):
        rewards, done, _ = _episode_data(11, E, Np, seed=k)
        all_returns.append(run.step(rewards, done))
    x = np.concatenate([a.reshape(-1) for a in all_returns]).astype(np.float64)
    n, mean, m2 = run.stats
    assert n == x.size
    np.testing.assert_allclose(mean[0], x.mean(), rtol=1e-12)
    np.testing.assert_allclose(m2[0] / n, x.var(), rtol=1e-10)
    scale = run.scale()
    assert scale.dtype == np.float32 and scale[0] == np.float32(1 / np.sqrt(m2[0] / n + 1e-8))
    y = scale_f32(rewards, scale, clip)
    assert np.array_equal(y, np.clip(np.multiply(rewards, scale[0], dtype=np.float32),
                                     -np.float32(clip), np.float32(clip)))
    run.reset()
    assert not run.carry.any()


# ------------------------------------------------------------------------ keys / refusals
def test_settings_and_their_refusals():
    from warp_drive_b200.training.reward_scale import reward_scale_settings

    assert reward_scale_settings({}, "p") == (False, 10.0)
    assert reward_scale_settings({"scale_rewards": False}, "p") == (False, 10.0)
    assert reward_scale_settings({"scale_rewards": True}, "p") == (True, 10.0)
    assert reward_scale_settings({"scale_rewards": True, "reward_clip": 5}, "p") == (True, 5.0)
    for bad in (1, "yes", None, 0.0):
        with pytest.raises(ValueError, match="scale_rewards is true or false"):
            reward_scale_settings({"scale_rewards": bad}, "p")
    with pytest.raises(ValueError, match="reward_clip needs scale_rewards: true"):
        reward_scale_settings({"reward_clip": 5.0}, "p")
    with pytest.raises(ValueError, match="reward_clip needs scale_rewards: true"):
        reward_scale_settings({"scale_rewards": False, "reward_clip": 5.0}, "p")
    for clip in (0, -1.0, float("inf"), float("nan"), True, False, "5", None):
        with pytest.raises(ValueError, match="reward_clip is a finite number > 0"):
            reward_scale_settings({"scale_rewards": True, "reward_clip": clip}, "p")


@pytest.mark.parametrize("trainer", ["TrainerDDPG", "TrainerTD3", "TrainerSAC", "TrainerDQN"])
@pytest.mark.parametrize("key,value", [("scale_rewards", True), ("reward_clip", 5.0)])
def test_replay_trainers_refuse_the_keys(trainer, key, value):
    from warp_drive_b200.training.trainer_ddpg import TrainerDDPG
    from warp_drive_b200.training.trainer_dqn import TrainerDQN
    from warp_drive_b200.training.trainer_sac import TrainerSAC
    from warp_drive_b200.training.trainer_td3 import TrainerTD3

    cls = {"TrainerDDPG": TrainerDDPG, "TrainerTD3": TrainerTD3, "TrainerSAC": TrainerSAC,
           "TrainerDQN": TrainerDQN}[trainer]
    model = ({"type": "fully_connected_q"} if trainer == "TrainerDQN"
             else {"actor": {"type": "fully_connected_actor"}, "critic": {}})
    config = {"policy": {"shared": {"model": model, key: value}},
              "sampler": {"params": {"epsilon": 0.1}}}
    with pytest.raises(ValueError, match=f"{trainer} does not take {key}"):
        cls(env_wrapper=None, config=config)


def _load(path):
    import yaml

    with open(path, encoding="utf8") as fp:
        return yaml.safe_load(fp)


def test_existing_configs_load_without_the_keys():
    from warp_drive_b200.training.reward_scale import reward_scale_settings

    paths = [p for p in sorted(glob.glob(os.path.join(CONFIGS, "*.yaml")))
             if not p.endswith("default_configs.yaml")]      # (its policy is not keyed by name)
    assert len(paths) > 20
    for path in paths:
        cfg = _load(path)
        for policy, pc in cfg.get("policy", {}).items():
            on = os.path.basename(path) == "single_pendulum_ppo_scaled.yaml"
            assert reward_scale_settings(pc, policy) == (on, 10.0), path


def test_scaled_pendulum_config_is_the_gae_config_with_both_normalizations():
    gae = _load(os.path.join(CONFIGS, "single_pendulum_ppo_gae.yaml"))
    scaled = _load(os.path.join(CONFIGS, "single_pendulum_ppo_scaled.yaml"))
    gae["policy"]["shared"]["scale_rewards"] = True
    gae["policy"]["shared"]["model"]["normalize_observations"] = True
    for d in (gae, scaled):
        d.pop("name")
        d["saving"].pop("name")
    assert scaled == gae


def test_buffers_are_the_identity():
    import torch
    from torch import nn

    from warp_drive_b200.training.reward_scale import register_buffers

    m = nn.Linear(2, 2)
    plain = list(m.state_dict())
    register_buffers(m)
    sd = m.state_dict()
    assert list(sd)[:len(plain)] == plain
    assert list(sd)[len(plain):] == ["return_count", "return_mean", "return_m2",
                                     "return_shift", "return_scale"]
    assert sd["return_count"].dtype == torch.float64 and sd["return_count"].shape == ()
    assert sd["return_mean"].dtype == sd["return_m2"].dtype == torch.float64
    assert sd["return_shift"].dtype == sd["return_scale"].dtype == torch.float32
    assert all(sd[k].shape == (1,) for k in ("return_mean", "return_m2", "return_shift",
                                              "return_scale"))
    assert float(sd["return_shift"]) == 0 and float(sd["return_scale"]) == 1
    assert [n for n, _ in m.named_parameters()] == ["weight", "bias"]


# ------------------------------------------------------------------------ C interface
def test_c_interface_and_ctypes_mirror():
    from warp_drive_b200 import lib as wlib

    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    i, vp, f = ctypes.c_int, ctypes.c_void_p, ctypes.c_float
    assert wlib._SIGNATURES["wdb_discounted_return_scan"] == (
        i, [vp, vp, vp, i, i, i, f, vp, vp])
    assert re.search(r"\bint wdb_discounted_return_scan\(void \*stream, const float \*rewards, "
                     r"const int \*done, int T,\s+int n_envs, int n_agents, float gamma, "
                     r"float \*carry,\s+float \*returns\);", header)


# ------------------------------------------------------------------------ ptxas
@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_scan_kernel_compiles_without_spills_or_fma(tmp_path):
    out = str(tmp_path / "rs.cubin")
    proc = subprocess.run(
        ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler",
         "-fPIC", "-Xptxas", "-v", "-cubin",
         os.path.join(ROOT, "warp_drive_b200", "csrc", "wdb_reward_scale.cu"), "-o", out],
        capture_output=True, text=True, check=True)
    entries = re.findall(r"Compiling entry function '(\w+)'", proc.stderr)
    assert len(entries) == 1 and "discounted_return_scan_kernel" in entries[0], entries
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", proc.stderr)
    assert spills and all(s == ("0", "0") for s in spills), spills
    if shutil.which("cuobjdump"):
        sass = subprocess.run(["cuobjdump", "-sass", out], capture_output=True, text=True,
                              check=True).stdout
        assert "FMUL" in sass and "FADD" in sass and "FFMA" not in sass
