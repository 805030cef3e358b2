#!/usr/bin/env python
"""Learning probe of the replay buffer: single_pendulum_{ddpg,td3,sac}_replay.yaml against
single_pendulum.yaml (DDPG over the ring of one rollout) at the same number of envs, the same
seed and the same number of env steps; prints one JSON object with each run's mean episodic
reward (training episodes, with each algorithm's own exploration) at the same env-step
checkpoints and its wall time.  A report, not a test: every Pendulum step costs between 0
(upright and still) and about -16.3, so a swing-up policy's episodic reward climbs towards 0.

    python scripts/pendulum_replay_learning.py [--env-steps 20000000] [--checkpoints 8]
"""
import argparse
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CONFIGS = ("single_pendulum", "single_pendulum_ddpg_replay", "single_pendulum_td3_replay",
           "single_pendulum_sac_replay")


def run(config, envs, env_steps, checkpoints, basedir):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent.classic_control import CUDAClassicControlPendulumEnv
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_ddpg import TrainerDDPG
    from warp_drive_b200.training.trainer_sac import TrainerSAC
    from warp_drive_b200.training.trainer_td3 import TrainerTD3

    cfg = load_run_config(config)
    T = cfg["trainer"]["train_batch_size"] // cfg["trainer"]["num_envs"]
    per_iter = envs * T
    iters = env_steps // per_iter
    cfg["trainer"].update(num_envs=envs, train_batch_size=per_iter, seed=3,
                          num_episodes=iters * per_iter // cfg["env"]["episode_length"] + 1)
    cfg["env"]["reset_pool_size"] = envs
    cfg["saving"].update(basedir=basedir, metrics_log_freq=max(1, iters // checkpoints),
                         model_params_save_freq=10 ** 9)
    cls = {"DDPG": TrainerDDPG, "TD3": TrainerTD3, "SAC": TrainerSAC}[
        cfg["policy"]["shared"]["algorithm"]]
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
            # a logging iteration in which no episode ended reports 0 steps: not a checkpoint
            if "Mean episodic reward" in m and m.get("Mean episodic steps", 0) > 0:
                curve.append((rec["Iterations Completed"] * per_iter,
                              round(m["Mean episodic reward"], 1)))
    updates = 1 if tr.replay is None else tr.replay["updates"]
    return {"iterations": tr.num_iters, "envs": envs, "env_steps_per_iteration": per_iter,
            "updates_per_iteration": updates, "rows_per_update": tr.fused_updates["shared"].rows,
            "wall_s": round(wall, 1), "mean_episodic_reward_at_env_steps": curve}


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=256)
    ap.add_argument("--env-steps", type=int, default=20000000)
    ap.add_argument("--checkpoints", type=int, default=8)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("pendulum_replay_learning.py needs a GPU")
    out = {}
    with tempfile.TemporaryDirectory() as basedir:
        for config in CONFIGS:
            out[config] = run(config, a.envs, a.env_steps, a.checkpoints, basedir)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
