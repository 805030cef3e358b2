#!/usr/bin/env python
"""Learning probe of TQC: single_pendulum_tqc_replay.yaml against single_pendulum_sac_replay.yaml
(the same sizes, replay buffer and actor) at the same number of envs and env steps, over several
seeds; prints one JSON object with each run's mean episodic training reward at the same env-step
checkpoints and its wall time.  A report, not a test: every Pendulum step costs between 0
(upright and still) and about -16.3, so a swing-up policy's episodic reward climbs towards 0.

    python scripts/pendulum_tqc_learning.py [--env-steps 10000000] [--seeds 1 2 3]
"""
import argparse
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CONFIGS = {"TQC": "single_pendulum_tqc_replay", "SAC": "single_pendulum_sac_replay"}


def run(algo, seed, envs, env_steps, checkpoints, basedir):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent.classic_control import CUDAClassicControlPendulumEnv
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_sac import TrainerSAC
    from warp_drive_b200.training.trainer_tqc import TrainerTQC

    cfg = load_run_config(CONFIGS[algo])
    T = cfg["trainer"]["train_batch_size"] // cfg["trainer"]["num_envs"]
    per_iter = envs * T
    iters = env_steps // per_iter
    cfg["trainer"].update(num_envs=envs, train_batch_size=per_iter, seed=seed,
                          num_episodes=iters * per_iter // cfg["env"]["episode_length"] + 1)
    cfg["env"]["reset_pool_size"] = envs
    cfg["saving"].update(basedir=basedir, metrics_log_freq=max(1, iters // checkpoints),
                         model_params_save_freq=10 ** 9)
    cls = TrainerTQC if algo == "TQC" else TrainerSAC
    w = EnvWrapper(CUDAClassicControlPendulumEnv(**cfg["env"]), num_envs=envs,
                   env_backend="numba")
    tr = cls(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
             results_dir=f"{algo}_{seed}", verbose=False)
    assert "shared" in tr.fused_updates and tr.engine.sa is not None
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
    return {"iterations": tr.num_iters, "wall_s": round(wall, 1),
            "mean_episodic_reward_at_env_steps": curve}


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=256)
    ap.add_argument("--env-steps", type=int, default=10000000)
    ap.add_argument("--checkpoints", type=int, default=4)
    ap.add_argument("--seeds", type=int, nargs="+", default=[1, 2, 3])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("pendulum_tqc_learning.py needs a GPU")
    out = {"envs": a.envs, "env_steps": a.env_steps}
    with tempfile.TemporaryDirectory() as basedir:
        for seed in a.seeds:
            for algo in CONFIGS:
                out[f"{algo} seed {seed}"] = run(algo, seed, a.envs, a.env_steps,
                                                 a.checkpoints, basedir)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
