#!/usr/bin/env python
"""Cost of running reward scaling (policy key scale_rewards), rounds alternated in one process:
  * the scaling one policy's update runs per iteration (RewardScaler.scale: the scan, the two
    moments launches and the scaling; four launches) and the scan alone, at 10 000 envs x
    T = 10 x 1 agent = 1e5 rows (single_pendulum_ppo_gae.yaml's batch) and at config 2's
    runner policy, 2 000 envs x T = 10 x 100 agents (bench.py --mode train);
  * ms per training iteration (rollout + update, not a logging iteration) of
    single_pendulum_ppo_gae.yaml with and without scale_rewards.
CUDA events around many calls; median and min-max over the rounds, and the GPU name and power
limit read in the same run.  Prints one JSON object.

    python scripts/bench_reward_scale.py [--rounds 7] [--reps 50] [--iters 10]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
from torch import nn  # noqa: E402

from warp_drive_b200 import lib as wlib  # noqa: E402
from warp_drive_b200.training import reward_scale  # noqa: E402


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def summary(xs):
    xs = sorted(xs)
    return {"median": xs[len(xs) // 2], "min": xs[0], "max": xs[-1], "n": len(xs)}


def scaling_cases(T, E, Np):
    g = torch.Generator(device="cuda").manual_seed(T + E + Np)
    rewards = torch.randn((T, E, Np), device="cuda", generator=g) * 4 - 8
    done = (torch.rand((T, E), device="cuda", generator=g) < 0.01).to(torch.int32)
    model = nn.Module()
    reward_scale.register_buffers(model)
    model.cuda()
    scaler = reward_scale.RewardScaler(model, (T, E, Np), 0.95, 10.0, "cuda")
    L = wlib.load()

    def scan():
        wlib.check(L.wdb_discounted_return_scan(
            wlib.stream_ptr(), wlib.ptr(rewards), wlib.ptr(done), T, E, Np, scaler.gamma,
            wlib.ptr(scaler.carry), wlib.ptr(scaler.returns)), "scan")

    return {"scale": lambda: scaler.scale(rewards, done), "scan": scan}


def pendulum_trainer(scaled, basedir):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent import classic_control as cc
    from warp_drive_b200.training.trainer import Trainer, load_run_config

    cfg = load_run_config("single_pendulum_ppo_gae")
    cfg["saving"].update(basedir=basedir, metrics_log_freq=10 ** 6, model_params_save_freq=10 ** 6)
    if scaled:
        cfg["policy"]["shared"]["scale_rewards"] = True
    env = cc.CUDAClassicControlPendulumEnv(**cfg["env"])
    wrapper = EnvWrapper(env, num_envs=cfg["trainer"]["num_envs"], env_backend="numba")
    tr = Trainer(env_wrapper=wrapper, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                 results_dir=f"scaled_{scaled}", verbose=False)
    assert tr.engine.sa is not None and bool(tr._reward_scalers) == scaled
    return tr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--iters", type=int, default=10, help="training iterations per round")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    out = {"gpu": gpu_info()}

    shapes = {"pendulum 10000 x T10 x 1": (10, 10_000, 1),
              "config 2 runner 2000 x T10 x 100": (10, 2_000, 100)}
    cases = {f"{what} {name}": fn for name, shape in shapes.items()
             for what, fn in scaling_cases(*shape).items()}
    for fn in cases.values():
        fn()
    res = {k: [] for k in cases}
    for _ in range(args.rounds):
        for k, fn in cases.items():
            res[k].append(timed(fn, args.reps) * 1e3)
    out["us_per_call"] = {k: summary(v) for k, v in res.items()}

    with tempfile.TemporaryDirectory() as basedir:
        trainers = {s: pendulum_trainer(s, basedir) for s in (False, True)}
        it = {s: 1 for s in trainers}

        def iteration(s):
            tr = trainers[s]
            tr._generate_rollout_batch()
            tr._update_model_params(it[s])          # never a logging iteration
            it[s] += 1

        for s in trainers:
            for _ in range(3):
                iteration(s)
        torch.cuda.synchronize()
        iters = {"plain": [], "scale_rewards": []}
        for _ in range(args.rounds):
            for s, name in ((False, "plain"), (True, "scale_rewards")):
                iters[name].append(timed(lambda s=s: iteration(s), args.iters))
        out["pendulum_ppo_gae_ms_per_iteration"] = {k: summary(v) for k, v in iters.items()}
        tr = trainers[False]
        out["iteration_shape"] = {"envs": tr.num_envs, "T": tr.engine.T,
                                  "optimizer_steps": tr._minibatch_steps}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
