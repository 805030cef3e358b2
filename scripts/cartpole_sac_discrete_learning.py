"""CartPole: discrete-action SAC (single_cartpole_sac_discrete.yaml) against double DQN
(single_cartpole_dqn.yaml) at the same env steps, over a few seeds.  After training, every env
plays one greedy episode with the evaluator (SAC: argmax pi; DQN: epsilon = 0); the episode cap
is 500 steps.  Prints a Markdown table and one JSON line, with the card name and power limit.

    python scripts/cartpole_sac_discrete_learning.py [--env-steps 2000000] [--envs 256]
                                                     [--seeds 1 2 3]
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

CONFIGS = {"discrete SAC": "single_cartpole_sac_discrete", "DQN": "single_cartpole_dqn"}


def run(algo, env_steps, envs, seed):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent.cartpole import CUDAClassicControlCartPoleEnv
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_dqn import TrainerDQN
    from warp_drive_b200.training.trainer_sac_discrete import TrainerDiscreteSAC

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
    cls = TrainerDiscreteSAC if algo == "discrete SAC" else TrainerDQN
    tr = cls(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
             results_dir=f"{algo.replace(' ', '_')}_{seed}", verbose=False)
    torch.cuda.synchronize()
    t0 = time.time()
    tr.train()
    torch.cuda.synchronize()
    wall = time.time() - t0
    greedy = {"use_argmax": True} if algo == "discrete SAC" else {"epsilon": 0}
    _, steps = tr.evaluate_episodes(**greedy)
    steps = steps["shared"].float()
    out = {"algorithm": algo, "seed": seed, "native_update": "shared" in tr.fused_updates,
           "one_launch_rollout": tr.engine.sa is not None,
           "env_steps": tr.num_iters * tr.training_batch_size, "wall_s": wall,
           "greedy_episode_steps_mean": float(steps.mean()),
           "greedy_episode_steps_min": float(steps.min()),
           "envs_at_cap": float((steps >= ep).float().mean())}
    if algo == "discrete SAC":
        out["alpha"] = float(tr.temperatures["shared"].log_alpha.detach().exp())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--env-steps", type=int, default=2_000_000)
    ap.add_argument("--envs", type=int, default=256)
    ap.add_argument("--seeds", type=int, nargs="*", default=[1, 2, 3])
    ap.add_argument("--only", nargs="*", default=list(CONFIGS), help="a subset of the runs")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rows = [run(a, args.env_steps, args.envs, s) for a in CONFIGS if a in args.only
            for s in args.seeds]
    print(f"{gpu}; {args.envs} envs")
    print("| algorithm | seed | env steps | wall (s) | greedy episode steps: mean | min "
          "| share at 500 |")
    print("|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['algorithm']} | {r['seed']} | {r['env_steps']} | {r['wall_s']:.1f} | "
              f"{r['greedy_episode_steps_mean']:.1f} | {r['greedy_episode_steps_min']:.0f} | "
              f"{r['envs_at_cap']:.2f} |")
    print(json.dumps({"gpu": gpu, "envs": args.envs, "runs": rows}))


if __name__ == "__main__":
    main()
