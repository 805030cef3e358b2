#!/usr/bin/env python
"""TD3 update at the single_pendulum_td3.yaml sizes (10 000 envs, T = 5, n_step 5, [64, 64]
actor and twin critics): ms per critic-only update and per actor update (TrainerTD3.
_update_model_params on a full ring, not a logging iteration) and per full iteration (rollout +
update, the actor stepping every other one) of the fused path (wdb_td3_critic_update /
wdb_td3_actor_update + FlatAdam) and of the torch autograd path, alternated in one process on
the same trainer and identical ring contents; libwdb200 launches per update; the achieved FLOP/s
of the fused updates from FLOP counts computed from the shapes; the GPU name and power limit.
Prints one JSON object."""
import json
import os
import sys
import tempfile

_HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(_HERE))
sys.path.insert(0, _HERE)

import torch  # noqa: E402

from bench_ddpg_update import gpu_info, timed  # noqa: E402
from warp_drive_b200 import lib as wlib  # noqa: E402


def build(basedir):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent.classic_control import CUDAClassicControlPendulumEnv
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_td3 import TrainerTD3

    cfg = load_run_config("single_pendulum_td3")
    cfg["trainer"]["seed"] = 7
    cfg["saving"]["basedir"] = basedir
    E = cfg["trainer"]["num_envs"]
    w = EnvWrapper(CUDAClassicControlPendulumEnv(**cfg["env"]), num_envs=E, env_backend="numba")
    tr = TrainerTD3(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                    results_dir="bench", verbose=False)
    assert "shared" in tr.fused_updates, "the fused update is not selected"
    return tr


def _macs(ins, dims, out):
    w = [ins] + list(dims) + [out]
    return [w[i] * w[i + 1] for i in range(len(w) - 1)]


def critic_flops(F, A, actor_dims, critic_dims, loss_rows):
    """Multiply-adds x 2 of the critic pass: per loss row the target actor, both target
    critics and both critics forward, then both critics' input gradients (every layer but the
    first) and weight gradients."""
    a, c = _macs(F, actor_dims, A), _macs(F + A, critic_dims, 1)
    return 2.0 * loss_rows * (sum(a) + 4 * sum(c) + 2 * sum(c[1:]) + 2 * sum(c))


def actor_flops(F, A, actor_dims, critic_dims, loss_rows):
    """Multiply-adds x 2 of the actor pass: per loss row the actor and Q1 forward, Q1's input
    gradients (every layer but the first, plus the first's action columns), the actor's input
    gradients (every layer but the first) and weight gradients."""
    a, c = _macs(F, actor_dims, A), _macs(F + A, critic_dims, 1)
    return 2.0 * loss_rows * (sum(a) + sum(c) + sum(c[1:]) + A * critic_dims[0] + sum(a[1:])
                              + sum(a))


def main():
    with tempfile.TemporaryDirectory() as basedir:
        tr = build(basedir)
        algo = tr.trainers["shared"]
        actor = tr.actor_models["shared"]
        critic = tr.critic_models["shared"]
        fused = tr.fused_updates["shared"]
        delay = algo.policy_delay
        for _ in range(2):
            tr._generate_rollout_batch()
        assert tr.engine.isfull()
        paths = {"fused": True, "torch": False}

        def update(actor_step):
            # the next update is number `delay` (an actor update) or 1 (critic only)
            tr.update_count["shared"] = delay - 1 if actor_step else 0
            tr._update_model_params(1)          # never a logging iteration (freq 1000)

        def iteration():
            tr._generate_rollout_batch()
            tr._update_model_params(1)

        res = {"workload": f"single_pendulum_td3.yaml: {tr.num_envs} envs, T = {tr.engine.T}, "
                           f"n_step {tr.n_step}, actor {actor.fc_dims}, critics "
                           f"{critic.fc_dims}, policy_delay {delay}"}
        kinds = {"critic_update": False, "actor_update": True}
        for name, flag in paths.items():        # warm-up, launch counts
            algo.use_fused_update = flag
            res[name] = {}
            for kind, actor_step in kinds.items():
                for _ in range(3):
                    update(actor_step)
                torch.cuda.synchronize()
                c0 = wlib.launch_count()
                update(actor_step)
                torch.cuda.synchronize()
                res[name][f"libwdb200_launches_per_{kind}"] = wlib.launch_count() - c0
        samples = {n: {k: [] for k in list(kinds) + ["iter"]} for n in paths}
        for _ in range(7):                      # alternate the two paths
            for name, flag in paths.items():
                algo.use_fused_update = flag
                for kind, actor_step in kinds.items():
                    samples[name][kind].append(timed(lambda: update(actor_step), 20))
                samples[name]["iter"].append(timed(iteration, 10))
        algo.use_fused_update = True
        med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
        for name in paths:
            for key in samples[name]:
                label = "ms_per_iteration" if key == "iter" else f"ms_per_{key}"
                v = samples[name][key]
                res[name][label] = med(v)
                res[name][label + "_min_max"] = [min(v), max(v)]
        shape = (int(actor.flattened_obs_size), int(actor.output_dims[0]), actor.fc_dims,
                 critic.fc_dims, fused.rows)
        cf, af = critic_flops(*shape), actor_flops(*shape)
        res["critic_update_gflop"] = cf / 1e9
        res["actor_update_gflop"] = (cf + af) / 1e9
        for kind, flops in (("critic_update", cf), ("actor_update", cf + af)):
            res[f"fused_{kind}_tflops_achieved"] = (
                flops / (res["fused"][f"ms_per_{kind}"] * 1e-3) / 1e12)
            res[f"{kind}_speedup"] = res["torch"][f"ms_per_{kind}"] / res["fused"][f"ms_per_{kind}"]
        res["iteration_speedup"] = (res["torch"]["ms_per_iteration"]
                                    / res["fused"]["ms_per_iteration"])
        res["gpu"], res["power_limit"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
