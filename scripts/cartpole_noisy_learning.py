"""CartPole: noisy DQN and Rainbow against their epsilon-greedy counterparts, one run each, at the
same env steps and seed: single_cartpole_dqn.yaml, single_cartpole_noisy_dqn.yaml (the same
network with a noisy output layer and epsilon 0), single_cartpole_dueling_c51.yaml and
single_cartpole_rainbow.yaml (the same network with noisy streams and epsilon 0).  After
training, every env plays one greedy episode (epsilon = 0, the mean network) with the evaluator;
the episode cap is 500 steps.  One seed: it says nothing about the spread between seeds.  Prints
a Markdown table and one JSON line, with the card name and power limit.

    python scripts/cartpole_noisy_learning.py [--env-steps 4000000] [--envs 256] [--seed 7]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CONFIGS = {"DQN": "single_cartpole_dqn", "noisy DQN": "single_cartpole_noisy_dqn",
           "dueling C51 + PER": "single_cartpole_dueling_c51",
           "Rainbow": "single_cartpole_rainbow"}


def run(algo, env_steps, envs, seed):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent.cartpole import CUDAClassicControlCartPoleEnv
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_dqn import TrainerDQN

    cfg = load_run_config(CONFIGS[algo])
    t = cfg["trainer"]
    per_env = t["train_batch_size"] // t["num_envs"]        # the config's rollout length
    t.update(num_envs=envs, train_batch_size=envs * per_env, seed=seed)
    ep = cfg["env"]["episode_length"]
    t["num_episodes"] = -(-env_steps // ep)
    cfg["saving"].update(basedir=tempfile.mkdtemp(), metrics_log_freq=10 ** 9,
                         model_params_save_freq=10 ** 9)
    env = CUDAClassicControlCartPoleEnv(**cfg["env"])
    w = EnvWrapper(env, num_envs=envs, env_backend="numba")
    tr = TrainerDQN(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                    results_dir=algo.replace(" ", "_"), verbose=False)
    torch.cuda.synchronize()
    t0 = time.time()
    tr.train()
    torch.cuda.synchronize()
    wall = time.time() - t0
    _, steps = tr.evaluate_episodes(epsilon=0)
    steps = steps["shared"].float()
    return {"algorithm": algo, "native_update": "shared" in tr.fused_updates,
            "one_launch_rollout": tr.engine.sa is not None,
            "noisy_sigma": (float(torch.cat([L.weight_sigma.detach().abs().flatten() for L in
                                             tr.q_models["shared"].noisy_layers()]).mean())
                            if tr.q_models["shared"].noisy else None),
            "env_steps": tr.num_iters * tr.training_batch_size,
            "iterations": tr.num_iters, "wall_s": wall,
            "greedy_episode_steps_mean": float(steps.mean()),
            "greedy_episode_steps_min": float(steps.min()),
            "envs_at_cap": float((steps >= ep).float().mean())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--env-steps", type=int, default=4_000_000)
    ap.add_argument("--envs", type=int, default=256)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--only", nargs="*", default=list(CONFIGS), help="a subset of the runs")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rows = [run(a, args.env_steps, args.envs, args.seed) for a in CONFIGS if a in args.only]
    print(f"{gpu}; {args.envs} envs, seed {args.seed}")
    print("| algorithm | env steps | wall (s) | greedy episode steps: mean | min | share at 500 "
          "| mean abs sigma_W |")
    print("|---|---|---|---|---|---|---|")
    for r in rows:
        sigma = "-" if r["noisy_sigma"] is None else f"{r['noisy_sigma']:.4f}"
        print(f"| {r['algorithm']} | {r['env_steps']} | {r['wall_s']:.1f} | "
              f"{r['greedy_episode_steps_mean']:.1f} | {r['greedy_episode_steps_min']:.0f} | "
              f"{r['envs_at_cap']:.2f} | {sigma} |")
    print(json.dumps({"gpu": gpu, "envs": args.envs, "seed": args.seed, "runs": rows}))


if __name__ == "__main__":
    main()
