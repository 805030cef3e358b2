"""A recurrent Gaussian policy (fully_connected_gaussian_gru) against a feed-forward one
(fully_connected_gaussian) on ContinuousRecallEnv (tests/custom_env/continuous_recall_env*): a
cue on the circle of radius 0.8 is shown once and the last step of the 4-step episode pays
minus the distance of the action to it, so a memoryless policy cannot expect more than -0.8.
Both train with PPO from the same seed; each one's mean last-step reward over 20 more rollouts
with the trained policy sampling its actions is printed as one JSON line and written under --out.

    python scripts/continuous_recall_gru_learning.py [--iterations 300] [--out DIR]"""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "custom_env"))

MODELS = {"fully_connected_gaussian_gru": {"type": "fully_connected_gaussian_gru",
                                           "fc_dims": [32], "gru_dim": 32,
                                           "log_std_init": -0.5},
          "fully_connected_gaussian": {"type": "fully_connected_gaussian", "fc_dims": [32, 32],
                                       "log_std_init": -0.5}}


def last_step_reward(trainer, rollouts=20):
    """The mean reward per (env, agent) episode over `rollouts` more rollouts: every step but
    the last pays 0, so this is the mean last-step reward."""
    import torch

    eng = trainer.engine
    eng.episodic_reward_sum["shared"].zero_()
    eng.num_completed_episodes.zero_()
    for _ in range(rollouts):
        eng.rollout()
    torch.cuda.synchronize()
    n_agents = len(eng.policy_map["shared"])
    return float(eng.episodic_reward_sum["shared"]) / (
        float(eng.num_completed_episodes) * n_agents)


def main():
    from continuous_recall_env import MEMORYLESS_BOUND, make_trainer

    ap = argparse.ArgumentParser()
    ap.add_argument("--iterations", type=int, default=300)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    result = {"env": "ContinuousRecallEnv", "episode_length": 4, "iterations": a.iterations,
              "seed": a.seed, "memoryless_bound": MEMORYLESS_BOUND}
    with tempfile.TemporaryDirectory() as tmp:
        for name, model in MODELS.items():
            tr = make_trainer(model, name, tmp, seed=a.seed, iterations=a.iterations)
            tr.train()
            result[name] = last_step_reward(tr)
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "continuous_recall_gru_learning.json"), "w",
                  encoding="utf8") as fp:
            fp.write(line + "\n")


if __name__ == "__main__":
    main()
