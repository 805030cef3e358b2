"""A recurrent policy (fully_connected_gru) against a feed-forward one (fully_connected) on
RecallEnv (tests/custom_env/recall_env*): the cue is shown once and the last step of the
4-step episode pays 1 for naming it, so a memoryless policy cannot beat 1/2.  Both train with
PPO from the same seed; each one's final success rate (the fraction of (env, agent) episodes
paid over 20 more rollouts with the trained policy sampling its actions) is printed as one JSON
line and written under --out.

    python scripts/recall_gru_learning.py [--iterations 300] [--out DIR]"""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "custom_env"))


def main():
    import torch
    from recall_env import make_trainer

    ap = argparse.ArgumentParser()
    ap.add_argument("--iterations", type=int, default=300)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    models = {"fully_connected_gru": {"type": "fully_connected_gru", "fc_dims": [32],
                                      "gru_dim": 32},
              "fully_connected": {"type": "fully_connected", "fc_dims": [32, 32]}}
    result = {"env": "RecallEnv", "episode_length": 4, "iterations": a.iterations,
              "seed": a.seed}
    with tempfile.TemporaryDirectory() as tmp:
        for name, model in models.items():
            tr = make_trainer(model, name, tmp, seed=a.seed, iterations=a.iterations)
            tr.train()
            eng = tr.engine
            eng.episodic_reward_sum["shared"].zero_()
            eng.num_completed_episodes.zero_()
            for _ in range(20):
                eng.rollout()
            torch.cuda.synchronize()
            n_agents = len(eng.policy_map["shared"])
            result[name] = float(eng.episodic_reward_sum["shared"]) / (
                float(eng.num_completed_episodes) * n_agents)
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "recall_gru_learning.json"), "w", encoding="utf8") as fp:
            fp.write(line + "\n")


if __name__ == "__main__":
    main()
