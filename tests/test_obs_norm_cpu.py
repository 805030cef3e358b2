"""CPU tests of observation normalization: the float64 Welford / Chan reference against NumPy's
mean and variance, the model keys and their refusals, the state_dict of models with and without
the key, the C interface and its ctypes mirror, and what ptxas makes of the new kernels (no
spills; the normalizing rollout kinds at the existing kinds' registers)."""
import ctypes
import os
import re
import shutil
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from obs_norm_reference import (  # noqa: E402
    batch_moments, chan, device_records, moments, normalize_f32, shift_scale, welford)

CSRC = os.path.join(ROOT, "warp_drive_b200", "csrc")
NVCC_SM90A = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC"]


# ------------------------------------------------------------------------ the reference
@pytest.mark.parametrize("rows,F", [(1, 1), (17, 3), (1000, 4), (5000, 63)])
def test_welford_and_chan_match_numpy(rows, F):
    rng = np.random.default_rng(rows * 100 + F)
    x = (rng.normal(size=(rows, F)) * rng.uniform(0.01, 50, F) + rng.uniform(-5, 5, F))
    x = x.astype(np.float32)
    x64 = x.astype(np.float64)
    mean, var = x64.mean(axis=0), x64.var(axis=0)
    for n, m, m2 in (welford(x), batch_moments(x), batch_moments(x, n_ranges=min(rows, 7))):
        assert n == rows
        np.testing.assert_allclose(m, mean, rtol=1e-12, atol=1e-12 * np.abs(x64).max())
        np.testing.assert_allclose(m2 / n, var, rtol=1e-10, atol=1e-300)
    # successive batches merged into a running state == the moments of their concatenation
    splits = np.array_split(x, 3)
    run = (0.0, np.zeros(F), np.zeros(F))
    for part in splits:
        run = chan(run, welford(part))
    np.testing.assert_allclose(run[1], mean, rtol=1e-12, atol=1e-12 * np.abs(x64).max())
    np.testing.assert_allclose(run[2] / run[0], var, rtol=1e-10, atol=1e-300)


def test_empty_side_and_identity_before_samples():
    one = moments(np.ones((3, 2), np.float32) * 2)
    empty = (0.0, np.zeros(2), np.zeros(2))
    assert chan(empty, one) is one and chan(one, empty) is one
    shift, scale = shift_scale(0.0, np.zeros(4), np.zeros(4))
    assert shift.dtype == np.float32 and scale.dtype == np.float32
    assert np.all(shift == 0) and np.all(scale == 1)
    shift, scale = shift_scale(*one)
    assert np.all(shift == 2) and np.all(scale == np.float32(1e4))


def test_normalize_reference_is_float32_subtract_multiply_clamp():
    x = np.array([[1e30, -1e30, 3.0, np.float32(0.1)]], np.float32)
    shift = np.array([1.0, 1.0, 2.5, 0.3], np.float32)
    scale = np.array([1.0, 1.0, 7.0, 3.0], np.float32)
    y = normalize_f32(x, shift, scale, 5.0)
    assert y.dtype == np.float32
    assert y[0, 0] == 5.0 and y[0, 1] == -5.0 and y[0, 2] == np.float32(3.5)
    assert y[0, 3] == np.float32(np.float32(np.float32(0.1) - np.float32(0.3)) * np.float32(3))
    assert device_records(1) == 1 and device_records(1025) == 2
    assert device_records(2_100_000) == 512


# ------------------------------------------------------------------------ keys / refusals
def test_settings_and_their_refusals():
    from warp_drive_b200.training.obs_norm import obs_norm_settings

    assert obs_norm_settings({}, "fully_connected") == (False, 10.0)
    assert obs_norm_settings({"normalize_observations": True}, "m") == (True, 10.0)
    assert obs_norm_settings({"normalize_observations": True, "observation_clip": 5}, "m") == (
        True, 5.0)
    with pytest.raises(ValueError, match="observation_clip needs model.normalize_observations"):
        obs_norm_settings({"observation_clip": 5.0}, "m")
    with pytest.raises(ValueError, match="observation_clip needs model.normalize_observations"):
        obs_norm_settings({"normalize_observations": False, "observation_clip": 5.0}, "m")
    for bad in (1, "yes", None):
        with pytest.raises(ValueError, match="normalize_observations is true or false"):
            obs_norm_settings({"normalize_observations": bad}, "m")
    for clip in (0, -1.0, float("inf"), float("nan"), True, "5"):
        with pytest.raises(ValueError, match="observation_clip is a finite number > 0"):
            obs_norm_settings({"normalize_observations": True, "observation_clip": clip}, "m")


@pytest.mark.parametrize("trainer", ["TrainerDDPG", "TrainerTD3", "TrainerSAC", "TrainerDQN"])
@pytest.mark.parametrize("key,value", [("normalize_observations", True),
                                       ("observation_clip", 5.0)])
def test_replay_trainers_refuse_the_keys(trainer, key, value):
    from warp_drive_b200.training.trainer_ddpg import TrainerDDPG
    from warp_drive_b200.training.trainer_dqn import TrainerDQN
    from warp_drive_b200.training.trainer_sac import TrainerSAC
    from warp_drive_b200.training.trainer_td3 import TrainerTD3

    cls = {"TrainerDDPG": TrainerDDPG, "TrainerTD3": TrainerTD3, "TrainerSAC": TrainerSAC,
           "TrainerDQN": TrainerDQN}[trainer]
    model = ({"type": "fully_connected_q", key: value} if trainer == "TrainerDQN"
             else {"actor": {"type": "fully_connected_actor", key: value}, "critic": {}})
    config = {"policy": {"shared": {"model": model}},
              "sampler": {"params": {"epsilon": 0.1}}}
    with pytest.raises(ValueError, match=f"{trainer} does not take model.{key}"):
        cls(env_wrapper=None, config=config)


# ------------------------------------------------------------------------ model / state_dict
def _stub_env(F=3, continuous=False):
    from warp_drive_b200.utils.spaces import Box, Discrete

    act = Box(-1, 1, shape=(1,)) if continuous else Discrete(3)
    inner = SimpleNamespace(observation_space={0: Box(-1, 1, shape=(F,))},
                            action_space={0: act})
    dm = SimpleNamespace(get_shape=lambda name: (4, 1, 1, F))
    return SimpleNamespace(env=inner, cuda_data_manager=dm, n_agents=1)


@pytest.mark.parametrize("model_type", ["fully_connected", "fully_connected_gaussian"])
def test_buffers_only_with_the_key(model_type):
    import torch

    from warp_drive_b200.training.models.fully_connected import ModelFactory

    cls = ModelFactory.create(model_type)
    env = _stub_env(continuous=model_type.endswith("gaussian"))

    def make(**kw):
        torch.manual_seed(0)
        return cls(env, dict({"type": model_type, "fc_dims": [8, 8]}, **kw), "shared",
                   {"shared": [0]})

    plain, on = make(), make(normalize_observations=True, observation_clip=4.0)
    off = make(normalize_observations=False)
    stats = {"obs_count", "obs_mean", "obs_m2", "obs_shift", "obs_scale"}
    assert not stats & set(plain.state_dict()) and not stats & set(off.state_dict())
    assert list(off.state_dict()) == list(plain.state_dict())
    assert set(on.state_dict()) == set(plain.state_dict()) | stats
    sd = on.state_dict()
    assert sd["obs_count"].dtype == torch.float64 and sd["obs_count"].shape == ()
    assert sd["obs_mean"].dtype == sd["obs_m2"].dtype == torch.float64
    assert sd["obs_shift"].dtype == sd["obs_scale"].dtype == torch.float32
    assert all(sd[k].shape == (3,) for k in stats - {"obs_count"})
    assert torch.all(sd["obs_shift"] == 0) and torch.all(sd["obs_scale"] == 1)
    assert on.observation_clip == 4.0 and not plain.normalize_observations
    # the parameters are the same: the statistics are buffers, not trained
    assert [n for n, _ in on.named_parameters()] == [n for n, _ in plain.named_parameters()]
    # normalizing models take neither the wgmma forward nor (the tanh head) the one-launch kind
    from warp_drive_b200.training.models.fused_forward import FusedPolicyForward

    assert not FusedPolicyForward.supported(on)


# ------------------------------------------------------------------------ C interface
def test_c_interface_and_ctypes_mirror():
    from warp_drive_b200 import lib as wlib

    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    i, ll, vp, f = ctypes.c_int, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_float
    want = {
        "wdb_obs_moments_scratch_doubles": (ll, [ll, i]),
        "wdb_obs_moments_update": (i, [vp, vp, ll, i, vp, vp, vp, vp, vp, vp]),
        "wdb_obs_moments_batch": (i, [vp, vp, ll, i, vp, vp]),
        "wdb_obs_moments_merge": (i, [vp, vp, i, i, vp, vp, vp, vp, vp]),
        "wdb_obs_normalize": (i, [vp, vp, vp, ll, i, vp, vp, f]),
    }
    for name, sig in want.items():
        assert wlib._SIGNATURES[name] == sig, name
        assert re.search(rf"\b{name}\(", header), name
    # the struct keeps its layout: the normalizing kinds read their arguments behind log_std
    fields = [n for n, _ in wlib.SaRollout._fields_]
    assert fields[-2:] == ["log_std", "gaussian_head"]
    assert "6 = softmax on normalized observations" in header


# ------------------------------------------------------------------------ ptxas
def _ptxas(src, tmp_path):
    out = str(tmp_path / (os.path.basename(src) + ".cubin"))
    proc = subprocess.run(NVCC_SM90A + ["-Xptxas", "-v", "-cubin", "-I",
                                        os.path.join(ROOT, "include"),
                                        os.path.join(CSRC, src), "-o", out],
                          capture_output=True, text=True, check=True)
    stats, name = {}, None
    for line in proc.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name = m.group(1)
            stats[name] = {}
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name and "spill" not in stats[name]:
            stats[name]["spill"] = (int(m.group(1)), int(m.group(2)))
        m = re.search(r"Used (\d+) registers", line)
        if m and name:
            stats[name]["regs"] = int(m.group(1))
    return stats


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_new_kernels_compile_without_spills(tmp_path):
    stats = _ptxas("wdb_obs_norm.cu", tmp_path)
    names = ("obs_moments_partial_kernel", "obs_moments_merge_kernel", "obs_normalize_kernel")
    for k in names:
        hits = [v for n, v in stats.items() if k in n]
        assert len(hits) == 1, (k, list(stats))
        assert hits[0]["spill"] == (0, 0), (k, hits[0])
    stats = _ptxas("wdb_sa_rollout_obs_norm.cu", tmp_path)
    kinds = {int(re.search(r"sa_rollout_kernelILi(\d)E", n).group(1)): v
             for n, v in stats.items() if "sa_rollout_kernel" in n}
    assert set(kinds) == {7, 8}
    for v in kinds.values():
        assert v["spill"] == (0, 0), kinds
        # the softmax and Gaussian kinds' budget: 10 CTAs of 64 threads per SM
        assert v["regs"] <= 96, kinds
