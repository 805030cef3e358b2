#!/usr/bin/env python
"""DDPG rollout at the single_pendulum.yaml sizes (10 000 envs, T = 5, n_step 5, reset pool
10 000, [64, 64] actor): ms per rollout timestep of the one-launch path
(wdb_single_agent_rollout) and of the generic per-step path (actor forward ->
wdb_sample_ou_process -> step -> bookkeeping -> reset), alternated in one process on the same
trainer and buffers; libwdb200 launches per rollout; ms per full TrainerDDPG iteration
(rollout + update) on each path; the GPU name and power limit.  Prints one JSON object."""
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from warp_drive_b200 import lib as wlib  # noqa: E402


def build(basedir):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent.classic_control import CUDAClassicControlPendulumEnv
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_ddpg import TrainerDDPG

    cfg = load_run_config("single_pendulum")
    cfg["trainer"]["seed"] = 7
    cfg["saving"]["basedir"] = basedir
    E = cfg["trainer"]["num_envs"]
    w = EnvWrapper(CUDAClassicControlPendulumEnv(**cfg["env"]), num_envs=E, env_backend="numba")
    tr = TrainerDDPG(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                     results_dir="bench", verbose=False)
    assert tr.engine.sa is not None, "the one-launch rollout is not selected"
    return tr


def gpu_info():
    name = torch.cuda.get_device_name()
    try:
        power = subprocess.run(
            ["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
             f"--id={torch.cuda.current_device()}"],
            capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    return name, power


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    with tempfile.TemporaryDirectory() as basedir:
        tr = build(basedir)
        eng = tr.engine
        sa, T = eng.sa, eng.T
        params = tr._get_sample_params()
        paths = {"fused": sa, "generic": None}
        iteration = [1]     # never a logging iteration (metrics_log_freq = 1000)

        def rollout():
            eng.rollout(**params)

        def train_iteration():
            tr._generate_rollout_batch()
            tr._update_model_params(iteration[0])

        res = {"workload": f"single_pendulum.yaml: {tr.num_envs} envs, T = {T}, "
                           f"n_step {tr.n_step}, reset pool 10000, actor [64, 64]"}
        for name, path in paths.items():            # warm-up, launch counts
            eng.sa = path
            for _ in range(3):
                train_iteration()
            torch.cuda.synchronize()
            # one full cycle of ring cursors: the one-launch path splits a rollout that wraps
            c0 = wlib.launch_count()
            for _ in range(eng.ring_capacity):
                rollout()
            torch.cuda.synchronize()
            res[name] = {"libwdb200_launches_per_rollout":
                         (wlib.launch_count() - c0) / eng.ring_capacity}
        samples = {n: {"step": [], "iter": []} for n in paths}
        for _ in range(5):                          # alternate the two paths
            for name, path in paths.items():
                eng.sa = path
                samples[name]["step"].append(timed(rollout, 50) / T)
                samples[name]["iter"].append(timed(train_iteration, 10))
        eng.sa = sa
        med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
        for name in paths:
            res[name]["ms_per_rollout_timestep"] = med(samples[name]["step"])
            res[name]["ms_per_rollout_timestep_spread"] = [min(samples[name]["step"]),
                                                           max(samples[name]["step"])]
            res[name]["ms_per_ddpg_iteration"] = med(samples[name]["iter"])
            res[name]["ms_per_ddpg_iteration_spread"] = [min(samples[name]["iter"]),
                                                         max(samples[name]["iter"])]
        res["rollout_speedup"] = (res["generic"]["ms_per_rollout_timestep"]
                                  / res["fused"]["ms_per_rollout_timestep"])
        res["iteration_speedup"] = (res["generic"]["ms_per_ddpg_iteration"]
                                    / res["fused"]["ms_per_ddpg_iteration"])
        res["gpu"], res["power_limit"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
