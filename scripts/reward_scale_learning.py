#!/usr/bin/env python
"""Learning probe: single_pendulum_ppo_gae.yaml raw, with scale_rewards, and with both
scale_rewards and model.normalize_observations (single_pendulum_ppo_scaled.yaml), on each seed
at the same envs and iterations (equal env steps); prints one JSON object with each run's mean
episodic reward (training episodes) at every logging iteration, its last reward scale and its
wall time.  A report, not a test.

    python scripts/reward_scale_learning.py [--iters 1000] [--seeds 1 2 3]
"""
import argparse
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

VARIANTS = {"raw": (False, False), "scale_rewards": (True, False), "both": (True, True)}


def run(variant, envs, iters, log_every, seed, basedir):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent import classic_control as cc
    from warp_drive_b200.training.trainer import Trainer, load_run_config

    scale, norm = VARIANTS[variant]
    cfg = load_run_config("single_pendulum_ppo_gae")
    T = cfg["trainer"]["train_batch_size"] // cfg["trainer"]["num_envs"]
    envs = envs or cfg["trainer"]["num_envs"]
    cfg["trainer"].update(num_envs=envs, train_batch_size=envs * T, seed=seed,
                          num_episodes=iters * envs * T // cfg["env"]["episode_length"])
    cfg["saving"].update(basedir=basedir, metrics_log_freq=log_every,
                         model_params_save_freq=10 ** 9)
    if scale:
        cfg["policy"]["shared"]["scale_rewards"] = True
    if norm:
        cfg["policy"]["shared"]["model"]["normalize_observations"] = True
    w = EnvWrapper(cc.CUDAClassicControlPendulumEnv(**cfg["env"]), num_envs=envs,
                   env_backend="numba")
    tr = Trainer(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                 results_dir=f"{variant}_{seed}", verbose=False)
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
    if scale:
        out["reward_scale"] = float(tr.models["shared"].return_scale)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=1000)
    ap.add_argument("--log-every", type=int, default=100)
    ap.add_argument("--seeds", type=int, nargs="+", default=[1, 2, 3])
    ap.add_argument("--envs", type=int, default=0, help="0: the config's num_envs")
    a = ap.parse_args()
    out = {}
    with tempfile.TemporaryDirectory() as basedir:
        for seed in a.seeds:
            for variant in VARIANTS:
                out[f"{variant} seed {seed}"] = run(variant, a.envs, a.iters, a.log_every, seed,
                                                    basedir)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
