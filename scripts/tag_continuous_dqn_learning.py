"""TagContinuous trained with branching DQN (tag_continuous_dqn.yaml), against random play.

For each seed: `--iterations` TrainerDQN iterations of the run config (each a 4-step rollout of
50 envs and 2 updates of 1024 windows per policy), then one greedy episode (epsilon 0) per env,
and one episode per env at epsilon 1 (every head uniform: the random baseline) from the same
trainer.  Prints one JSON line: per seed and policy the mean episodic reward per agent of both,
and the training curve: the mean per-agent episodic reward of the episodes the training rollouts
completed in each block of `--log-every` iterations.  Card name and power limit are read in the
same run.

    python scripts/tag_continuous_dqn_learning.py [--seeds 1 2 3] [--iterations 2500]
"""
import argparse
import json
import os
import sys
import tempfile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from bench_dqn import gpu_info  # noqa: E402


def make_trainer(seed):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.tag_continuous import TagContinuous
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_dqn import TrainerDQN

    cfg = load_run_config("tag_continuous_dqn")
    cfg["trainer"].update(seed=seed, evaluator=False)
    cfg["saving"].update(basedir=tempfile.mkdtemp(), metrics_log_freq=10 ** 9,
                         model_params_save_freq=10 ** 9)
    env = TagContinuous(**cfg["env"])
    w = EnvWrapper(env, num_envs=cfg["trainer"]["num_envs"], env_backend="b200")
    n_t, n_r = cfg["env"]["num_taggers"], cfg["env"]["num_runners"]
    pm = {"tagger": list(range(n_t)), "runner": list(range(n_t, n_t + n_r))}
    return TrainerDQN(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map=pm,
                      results_dir=f"learn{seed}", verbose=False)


def per_agent(rewards):
    return {p: round(float(r.double().mean()), 4) for p, r in rewards.items()}


def run(seed, iterations, log_every):
    tr = make_trainer(seed)
    assert set(tr.fused_updates) == {"tagger", "runner"}
    eng = tr.engine
    curve = []
    for it in range(iterations):
        tr._generate_rollout_batch()
        tr._update_model_params(it + 1)
        if (it + 1) % log_every == 0:
            done = max(int(eng.num_completed_episodes), 1)
            curve.append({"iteration": it + 1, **{
                p: round(float(eng.episodic_reward_sum[p]) / done / len(ids), 4)
                for p, ids in tr.policy_tag_to_agent_id_map.items()}})
            for p in tr.policies:
                eng.episodic_reward_sum[p].zero_()
            eng.num_completed_episodes.zero_()
    greedy, _ = tr.evaluate_episodes(epsilon=0.0)
    random, _ = tr.evaluate_episodes(epsilon=1.0)
    torch.cuda.synchronize()
    return {"seed": seed, "greedy": per_agent(greedy), "random": per_agent(random),
            "curve": curve}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, nargs="+", default=[1, 2, 3])
    ap.add_argument("--iterations", type=int, default=2500)
    ap.add_argument("--log-every", type=int, default=500)
    args = ap.parse_args()
    out = {"gpu": gpu_info(), "iterations": args.iterations,
           "runs": [run(s, args.iterations, args.log_every) for s in args.seeds]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
