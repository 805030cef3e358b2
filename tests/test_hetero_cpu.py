"""Heterogeneous-agent training without a GPU: the layout of the gather / bookkeeping structs
that gained per-policy sources, the step and batch placeholders of the example env
(tests/custom_env/hetero_env*) for separate placeholders and agent-last observations,
Trainer / TrainerDDPG argument checks, and the generic rollout kernels compiled without
spills."""
import ctypes
import os
import re
import shutil
import subprocess
import sys
import types

import numpy as np
import pytest

from test_abi_layout_cpu import _c_fields

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(HERE, "custom_env"))

STRUCTS = {
    "wdb_gather_field": "GatherField", "wdb_gather_fields_policy": "GatherFieldsPolicy",
    "wdb_gather_fields": "GatherFields", "wdb_bookkeep_policy": "BookkeepPolicy",
    "wdb_bookkeep": "Bookkeep",
}


def test_gather_and_bookkeep_structs_match_the_header(tmp_path):
    from warp_drive_b200 import lib as wlib

    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "wdb200.h"', "int main(void) {"]
    fields = {}
    for c_name in STRUCTS:
        fields[c_name] = _c_fields(header, c_name)
        lines.append(f'  printf("{c_name} size %zu\\n", sizeof({c_name}));')
        for f in fields[c_name]:
            lines.append(f'  printf("{c_name} {f} %zu\\n", offsetof({c_name}, {f}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)],
                   check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    got = {(s, f): int(v) for s, f, v in (line.split() for line in out.splitlines())}
    for c_name, py_name in STRUCTS.items():
        cls = getattr(wlib, py_name)
        assert ctypes.sizeof(cls) == got[(c_name, "size")], c_name
        assert [n for n, _ in cls._fields_] == fields[c_name], c_name
        for f in fields[c_name]:
            assert getattr(cls, f).offset == got[(c_name, f)], (c_name, f)
    # the extensions sit behind the fields existing callers set, zero = the old behaviour
    assert [n for n, _ in wlib.GatherField._fields_][-3:] == [
        "policy_mask", "own_rows", "agents_last"]
    assert [n for n, _ in wlib.BookkeepPolicy._fields_][-3:] == ["rewards", "actions", "n_heads"]


# ---------------------------------------------------------------- placeholders
def _wrapper(E=3, **env_kw):
    from hetero_env import HeteroEnv

    from warp_drive_b200.managers.data_manager import CUDADataManager
    from warp_drive_b200.utils.spaces import obs_dict_to_spaces

    env = HeteroEnv(**env_kw)
    env.observation_space = obs_dict_to_spaces(env.reset())
    dm = CUDADataManager(num_agents=env.num_agents, episode_length=env.episode_length,
                         num_envs=E, device="cpu")
    return types.SimpleNamespace(env=env, n_envs=E, n_agents=env.num_agents,
                                 env_backend="pycuda", cuda_data_manager=dm,
                                 obs_at_reset=env.reset)


def _push(w, separate, layout, T=4):
    from warp_drive_b200.training.utils.data_loader import create_and_push_data_placeholders

    create_and_push_data_placeholders(
        env_wrapper=w, policy_tag_to_agent_id_map=w.env.policy_tag_to_agent_id_map(),
        create_separate_placeholders_for_each_policy=separate,
        obs_dim_corresponding_to_num_agents=layout, training_batch_size_per_env=T)
    dm = w.cuda_data_manager
    return {k: (tuple(dm.get_shape(k)), dm.get_dtype(k)) for k in dm._device_data_via_torch
            if not k.endswith("_at_reset")}


@pytest.mark.parametrize("layout", ["first", "last"])
def test_separate_placeholders_of_the_hetero_env(layout):
    w = _wrapper(E=3, num_agents=5, worker_obs_layout=layout)
    got = _push(w, True, layout)
    wobs = (3, 4, 2, 3) if layout == "first" else (3, 2, 3, 4)
    one = (lambda *f: (3, 1) + f) if layout == "first" else (lambda *f: (3,) + f + (1,))
    want = {
        "observations_planner_state": (one(3), "float32"),
        "observations_planner_action_mask": (one(8), "int32"),
        "sampled_actions_planner": ((3, 1, 2), "int32"),
        "sampled_actions_0_planner": ((3, 1, 1), "int32"),
        "sampled_actions_1_planner": ((3, 1, 1), "int32"),
        "rewards_planner": ((3, 1), "float32"),
        "observations_workers": (wobs, "float32"),
        "sampled_actions_workers": ((3, 4, 1), "int32"),
        "rewards_workers": ((3, 4), "float32"),
        "processed_observations_batch_planner": ((4, 3, 1, 3), "float32"),
        "action_mask_batch_planner": ((4, 3, 1, 8), "float32"),
        "sampled_actions_batch_planner": ((4, 3, 1, 2), "int32"),
        "rewards_batch_planner": ((4, 3, 1), "float32"),
        "processed_observations_batch_workers": ((4, 3, 4, 6), "float32"),
        "sampled_actions_batch_workers": ((4, 3, 4, 1), "int32"),
        "rewards_batch_workers": ((4, 3, 4), "float32"),
        "done_flags_batch": ((4, 3), "int32"),
    }
    for k, v in want.items():
        assert got[k] == v, (k, got[k], v)
    for name in ("observations", "sampled_actions", "rewards", "action_mask_batch_workers"):
        assert name not in got
    # the agent-last array is numpy.moveaxis of the agent-first one
    dm = w.cuda_data_manager
    first = np.stack([w.env.reset()[a] for a in range(1, 5)])
    arr = dm.pull_data_from_device("observations_workers")[0]
    assert np.array_equal(arr, first if layout == "first" else np.moveaxis(first, 0, -1))


def test_shared_agent_last_placeholders_of_the_workers_only_env():
    w = _wrapper(E=2, num_agents=6, with_planner=False, worker_obs_layout="last")
    got = _push(w, False, "last")
    assert got["observations"] == ((2, 2, 3, 6), "float32")
    assert got["sampled_actions"] == ((2, 6, 1), "int32")
    assert got["processed_observations_batch_workers"] == ((4, 2, 6, 6), "float32")


def test_placeholders_refuse_what_cannot_be_shared():
    with pytest.raises(AssertionError, match="identical"):
        _push(_wrapper(num_agents=4), False, "first")          # planner and workers differ
    w = _wrapper(num_agents=4, with_planner=False)
    with pytest.raises(AssertionError):
        _push(w, True, "first")                                 # one policy: nothing to separate


def test_hetero_twin_starts_where_the_env_resets():
    from hetero_env import HeteroEnv, HeteroTwin, planner_mask

    env = HeteroEnv(num_agents=5, episode_length=3)
    obs = env.reset()
    twin = HeteroTwin(2, 5, 3)
    o = twin.observe()
    assert np.array_equal(o["workers"][1], np.stack([obs[a] for a in range(1, 5)]))
    assert np.array_equal(o["planner_state"][0], obs[0]["state"])
    assert np.array_equal(o["planner_mask"][0], obs[0]["action_mask"])
    # valid actions never count as invalid; the episode ends and restarts after 3 steps
    for _ in range(3):
        m = twin.observe()["planner_mask"]
        pa = np.stack([2 * m[:, 2], (m[:, 3:].sum(1) - 1)], -1)
        rew, done = twin.step(np.zeros((2, 4), np.int64), pa)
    assert twin.invalid == 0 and done.all() and (twin.level == 0).all()
    assert np.array_equal(planner_mask(np.array([0, 4]))[:, :3], [[0, 1, 1], [1, 1, 0]])


# ---------------------------------------------------------------- trainers
def test_trainer_accepts_both_observation_layouts():
    from warp_drive_b200.training.trainer import Trainer

    for layout in ("first", "last"):
        Trainer._check_obs_dim(layout)
    with pytest.raises(AssertionError):
        Trainer._check_obs_dim("middle")


def test_trainer_ddpg_refuses_separate_placeholders():
    from warp_drive_b200.training.trainer_ddpg import TrainerDDPG

    with pytest.raises(AssertionError, match="separate per-policy placeholders"):
        TrainerDDPG(env_wrapper=None, config={},
                    create_separate_placeholders_for_each_policy=True)


# ---------------------------------------------------------------- no spills
@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_generic_rollout_kernels_compile_without_spills(tmp_path):
    src = os.path.join(ROOT, "warp_drive_b200", "csrc", "wdb_rollout_generic.cu")
    proc = subprocess.run(
        ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "g.o")],
        capture_output=True, text=True, check=True)
    stats = {}
    name = None
    for line in proc.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name = m.group(1)
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                      line)
        if m and name:
            stats[name] = tuple(int(x) for x in m.groups())
    kernels = {k: v for k, v in stats.items()
               if any(s in k for s in ("gather_fields_kernel", "bookkeep_kernel",
                                       "gather_rows_kernel"))}
    assert len(kernels) == 3, stats
    for k, v in kernels.items():
        assert v == (0, 0, 0), (k, v)
