"""Config-2 rollout (bench.py's engine: 2000 TagContinuous envs x 105 agents, sampling wgmma
forwards + the fused env step, CUDA graph) as one env group and as two, alternated in one
process: ms per step of each round, then the median and min-max of each schedule.

    python scripts/bench_rollout_groups.py [--rounds 5] [--steps 200] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--envs", type=int, default=2000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    import bench

    assert torch.cuda.is_available(), "needs a GPU"
    T = 100
    assert args.steps % T == 0
    _, engine, _, _ = bench.build_engine(args.envs, seed=1234, graph_steps=T)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout
    times = {1: [], 2: []}

    def timed(n):
        engine._set_env_groups(n)
        for _ in range(4):                   # capture + warm replays
            engine.rollout()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.steps // T):
            engine.rollout()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.steps

    for _ in range(args.rounds):
        for n in (1, 2):
            times[n].append(timed(n))
    res = {"card": card.strip(), "envs": args.envs, "steps": args.steps}
    for n, ms in times.items():
        s = sorted(ms)
        res[f"groups_{n}"] = {"ms_per_step": ms, "median": s[len(s) // 2], "min": s[0],
                              "max": s[-1]}
    res["speedup_median"] = res["groups_1"]["median"] / res["groups_2"]["median"]
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "rollout_groups.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
