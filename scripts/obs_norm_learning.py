#!/usr/bin/env python
"""Learning probe: single_mountain_car.yaml against single_mountain_car_obs_norm.yaml (A2C), and
single_pendulum_ppo.yaml with and without model.normalize_observations (PPO), each pair at the
same seed, envs and iterations (equal env steps); prints one JSON object with each run's mean
episodic reward (training episodes) at every logging iteration, its last observation
statistics and its wall time.  A report, not a test: one seed does not rank the two.

    python scripts/obs_norm_learning.py [--iters 200] [--seed 3]
"""
import argparse
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def run(config, norm, envs, iters, log_every, seed, basedir):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent import classic_control as cc
    from warp_drive_b200.training.trainer import Trainer, load_run_config

    cfg = load_run_config(config)
    T = cfg["trainer"]["train_batch_size"] // cfg["trainer"]["num_envs"]
    envs = envs or cfg["trainer"]["num_envs"]
    cfg["trainer"].update(num_envs=envs, train_batch_size=envs * T, seed=seed,
                          num_episodes=iters * envs * T // cfg["env"]["episode_length"])
    cfg["saving"].update(basedir=basedir, metrics_log_freq=log_every,
                         model_params_save_freq=10 ** 9)
    model = cfg["policy"]["shared"]["model"]
    if norm:
        model["normalize_observations"] = True
    else:
        model.pop("normalize_observations", None)
        model.pop("observation_clip", None)
    name = "Pendulum" if "pendulum" in config else "MountainCar"
    w = EnvWrapper(getattr(cc, f"CUDAClassicControl{name}Env")(**cfg["env"]), num_envs=envs,
                   env_backend="numba")
    tr = Trainer(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                 results_dir=f"{config}_{norm}", verbose=False)
    assert tr.engine.sa is not None
    t0 = time.time()
    tr.train()
    wall = time.time() - t0
    curve = []
    with open(os.path.join(tr.save_dir, "results.json"), encoding="utf8") as fp:
        for line in fp:
            rec = json.loads(line)
            m = rec.get("shared", {})
            if "Mean episodic reward" in m:
                curve.append((rec["Iterations Completed"], round(m["Mean episodic reward"], 2)))
    out = {"iterations": tr.num_iters, "envs": envs, "T": T, "seed": seed,
           "wall_s": round(wall, 1), "mean_episodic_reward": curve}
    m = tr.models["shared"]
    if norm:
        out["obs_mean"] = [round(v, 4) for v in m.obs_mean.tolist()]
        out["obs_std"] = [round(v, 4) for v in (m.obs_m2 / m.obs_count).sqrt().tolist()]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--log-every", type=int, default=20)
    ap.add_argument("--seed", type=int, default=3)
    ap.add_argument("--envs", type=int, default=0, help="0: the config's num_envs")
    a = ap.parse_args()
    out = {}
    with tempfile.TemporaryDirectory() as basedir:
        for config, norm in (("single_mountain_car", False),
                             ("single_mountain_car_obs_norm", True),
                             ("single_pendulum_ppo", False), ("single_pendulum_ppo", True)):
            out[f"{config}{'+norm' if norm and 'obs_norm' not in config else ''}"] = run(
                config, norm, a.envs, a.iters, a.log_every, a.seed, basedir)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
