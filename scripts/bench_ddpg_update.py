#!/usr/bin/env python
"""DDPG update at the single_pendulum.yaml sizes (10 000 envs, T = 5, n_step 5, [64, 64] actor
and critic): ms per update (TrainerDDPG._update_model_params on a full ring, not a logging
iteration) and per full iteration (rollout + update) of the fused path (wdb_ddpg_update +
FlatAdam) and of the torch autograd path, alternated in one process on the same trainer and
identical ring contents; libwdb200 launches per update; the achieved FLOP/s of the fused update
from a FLOP count computed from the shapes; the GPU name and power limit.  Prints one JSON
object."""
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
    assert "shared" in tr.fused_updates, "the fused update is not selected"
    return tr


def update_flops(F, A, actor_dims, critic_dims, loss_rows):
    """Multiply-adds x 2 of one update: per loss row the target actor and target critic, the
    critic on (obs, actions), the actor and the critic on (obs, pi) forward; the backward of
    the critic on both paths (input gradients of every layer but the first, plus the action
    columns of the first on the pi path), of the actor (every layer but the first) and the
    weight gradients of the three backward passes."""
    def macs(ins, dims, out):
        w = [ins] + list(dims) + [out]
        return [w[i] * w[i + 1] for i in range(len(w) - 1)]

    a = macs(F, actor_dims, A)
    c = macs(F + A, critic_dims, 1)
    forward = 2 * sum(a) + 3 * sum(c)
    input_grads = 2 * sum(c[1:]) + sum(a[1:]) + A * critic_dims[0]
    weight_grads = 2 * sum(c) + sum(a)
    return 2.0 * loss_rows * (forward + input_grads + weight_grads)


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
        algo = tr.trainers["shared"]
        actor = tr.actor_models["shared"]
        critic = tr.critic_models["shared"]
        fused = tr.fused_updates["shared"]
        for _ in range(2):
            tr._generate_rollout_batch()
        assert tr.engine.isfull()
        paths = {"fused": True, "torch": False}

        def update():
            tr._update_model_params(1)          # never a logging iteration (freq 1000)

        def iteration():
            tr._generate_rollout_batch()
            tr._update_model_params(1)

        res = {"workload": f"single_pendulum.yaml: {tr.num_envs} envs, T = {tr.engine.T}, "
                           f"n_step {tr.n_step}, actor {actor.fc_dims}, critic {critic.fc_dims}"}
        for name, flag in paths.items():        # warm-up, launch counts
            algo.use_fused_update = flag
            for _ in range(3):
                update()
            torch.cuda.synchronize()
            c0 = wlib.launch_count()
            update()
            torch.cuda.synchronize()
            res[name] = {"libwdb200_launches_per_update": wlib.launch_count() - c0}
        samples = {n: {"update": [], "iter": []} for n in paths}
        for _ in range(7):                      # alternate the two paths
            for name, flag in paths.items():
                algo.use_fused_update = flag
                samples[name]["update"].append(timed(update, 20))
                samples[name]["iter"].append(timed(iteration, 10))
        algo.use_fused_update = True
        med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
        for name in paths:
            for key, label in (("update", "ms_per_update"), ("iter", "ms_per_iteration")):
                v = samples[name][key]
                res[name][label] = med(v)
                res[name][label + "_min_max"] = [min(v), max(v)]
        flops = update_flops(int(actor.flattened_obs_size), int(actor.output_dims[0]),
                             actor.fc_dims, critic.fc_dims, fused.rows)
        res["fused_update_gflop"] = flops / 1e9
        res["fused_update_tflops_achieved"] = flops / (res["fused"]["ms_per_update"] * 1e-3) / 1e12
        res["update_speedup"] = res["torch"]["ms_per_update"] / res["fused"]["ms_per_update"]
        res["iteration_speedup"] = (res["torch"]["ms_per_iteration"]
                                    / res["fused"]["ms_per_iteration"])
        res["gpu"], res["power_limit"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
