#!/usr/bin/env python
"""Learning probe: single_pendulum.yaml (DDPG) and single_pendulum_td3.yaml (TD3) at a reduced
number of envs, the same seed and the same number of iterations; prints one JSON object with
each run's mean episodic reward (training episodes, with exploration noise) at every logging
iteration and its wall time.  A report, not a test: every Pendulum step costs between 0 (upright
and still) and about -16.3, so a swing-up policy's episodic reward climbs towards 0.

    python scripts/pendulum_td3_vs_ddpg.py [--envs 1024] [--iters 3000]
"""
import argparse
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def run(config, envs, iters, log_every, basedir):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent.classic_control import CUDAClassicControlPendulumEnv
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_ddpg import TrainerDDPG
    from warp_drive_b200.training.trainer_td3 import TrainerTD3

    cfg = load_run_config(config)
    T = cfg["trainer"]["train_batch_size"] // cfg["trainer"]["num_envs"]
    cfg["trainer"].update(num_envs=envs, train_batch_size=envs * T, seed=3,
                          num_episodes=iters * envs * T // cfg["env"]["episode_length"])
    cfg["env"]["reset_pool_size"] = envs
    cfg["saving"].update(basedir=basedir, metrics_log_freq=log_every,
                         model_params_save_freq=10 ** 9)
    cls = TrainerTD3 if cfg["policy"]["shared"]["algorithm"] == "TD3" else TrainerDDPG
    w = EnvWrapper(CUDAClassicControlPendulumEnv(**cfg["env"]), num_envs=envs,
                   env_backend="numba")
    tr = cls(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
             results_dir=config, verbose=False)
    assert "shared" in tr.fused_updates
    t0 = time.time()
    tr.train()
    wall = time.time() - t0
    curve = []
    with open(os.path.join(tr.save_dir, "results.json"), encoding="utf8") as fp:
        for line in fp:
            rec = json.loads(line)
            m = rec.get("shared", {})
            if "Mean episodic reward" in m:
                curve.append((rec["Iterations Completed"], round(m["Mean episodic reward"], 1)))
    return {"iterations": tr.num_iters, "envs": envs, "wall_s": round(wall, 1),
            "mean_episodic_reward": curve}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=3000)
    ap.add_argument("--log-every", type=int, default=250)
    a = ap.parse_args()
    out = {}
    with tempfile.TemporaryDirectory() as basedir:
        for config in ("single_pendulum", "single_pendulum_td3"):
            out[config] = run(config, a.envs, a.iters, a.log_every, basedir)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
