#!/usr/bin/env python
"""Cost of observation normalization (model.normalize_observations), rounds alternated in one
process:
  * the moments update (wdb_obs_moments_update, two launches) at 10 000 envs x T = 10 x F = 3
    (single_pendulum_ppo.yaml's batch) and at config 2's batch, 2 000 envs x 105 timesteps x 10
    agents = 2.1e6 rows of tag_continuous's observation width;
  * ms per rollout timestep of the one-launch rollout, with and without the key, for Pendulum
    Gaussian PPO (single_pendulum_ppo.yaml) and MountainCar A2C (single_mountain_car.yaml);
  * the per-step generic-path cost of wdb_obs_normalize on one step's observations (config 2's
    20 000 rows of each policy, and 10 000 rows x F = 3).
CUDA events around many launches; median and min-max over the rounds, and the GPU name and
power limit.  Prints one JSON object."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from warp_drive_b200 import lib as wlib  # noqa: E402


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


def tag_continuous_width():
    import yaml

    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.tag_continuous import TagContinuous
    from warp_drive_b200.training.utils.data_loader import get_flattened_obs_size

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "warp_drive_b200", "training", "run_configs",
                           "tag_continuous.yaml"), encoding="utf8") as fp:
        cfg = yaml.safe_load(fp)
    env = TagContinuous(**cfg["env"])
    w = EnvWrapper(env, num_envs=2, env_backend="b200")
    return int(get_flattened_obs_size(w.env.observation_space[0])), int(env.num_agents)


def moments_case(rows, F):
    L = wlib.load()
    x = torch.randn(rows, F, device="cuda") * 3 + 1
    scratch = torch.empty(int(L.wdb_obs_moments_scratch_doubles(rows, F)), dtype=torch.float64,
                          device="cuda")
    st = [torch.zeros((), dtype=torch.float64, device="cuda"),
          torch.zeros(F, dtype=torch.float64, device="cuda"),
          torch.zeros(F, dtype=torch.float64, device="cuda"),
          torch.zeros(F, device="cuda"), torch.ones(F, device="cuda")]

    def run():
        wlib.check(L.wdb_obs_moments_update(wlib.stream_ptr(), wlib.ptr(x), rows, F,
                                            wlib.ptr(scratch), *[wlib.ptr(t) for t in st]),
                   "update")
    return run, 2 * rows * F * 4


def normalize_case(rows, F):
    L = wlib.load()
    x = torch.randn(rows, F, device="cuda")
    y = torch.empty_like(x)
    shift, scale = torch.zeros(F, device="cuda"), torch.ones(F, device="cuda")

    def run():
        wlib.check(L.wdb_obs_normalize(wlib.stream_ptr(), wlib.ptr(x), wlib.ptr(y), rows, F,
                                       wlib.ptr(shift), wlib.ptr(scale), 10.0), "normalize")
    return run


def rollout_trainer(config, env_cls, norm, basedir):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent import classic_control as cc
    from warp_drive_b200.training.trainer import Trainer, load_run_config

    cfg = load_run_config(config)
    cfg["saving"].update(basedir=basedir, metrics_log_freq=10 ** 6, model_params_save_freq=10 ** 6)
    if norm:
        cfg["policy"]["shared"]["model"]["normalize_observations"] = True
    env = getattr(cc, env_cls)(**cfg["env"])
    wrapper = EnvWrapper(env, num_envs=cfg["trainer"]["num_envs"], env_backend="numba")
    tr = Trainer(env_wrapper=wrapper, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                 results_dir=f"{config}_{norm}", verbose=False)
    assert tr.engine.sa is not None and tr.engine.sa.normalizing == norm
    if norm:                                     # statistics that are not the identity
        tr._generate_rollout_batch()
        tr._update_observation_statistics()
    return tr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    out = {"gpu": gpu_info()}
    F_tag, n_agents = tag_continuous_width()
    out["tag_continuous_F"] = F_tag

    cases = {"moments 100000 x 3": moments_case(100_000, 3),
             f"moments 2100000 x {F_tag}": moments_case(2_100_000, F_tag)}
    norm = {"normalize 20000 x %d (config 2 step)" % F_tag: normalize_case(20_000, F_tag),
            "normalize 10000 x 3": normalize_case(10_000, 3)}
    for fn, _ in cases.values():
        fn()
    for fn in norm.values():
        fn()
    res = {k: [] for k in list(cases) + list(norm)}
    for _ in range(args.rounds):
        for k, (fn, _) in cases.items():
            res[k].append(timed(fn, args.reps) * 1e3)
        for k, fn in norm.items():
            res[k].append(timed(fn, args.reps * 4) * 1e3)
    out["us_per_call"] = {k: summary(v) for k, v in res.items()}
    out["moments_GBps_at_median"] = {
        k: nbytes / 2 / (out["us_per_call"][k]["median"] * 1e-6) / 1e9
        for k, (_, nbytes) in cases.items()}

    with tempfile.TemporaryDirectory() as basedir:
        pairs = {"pendulum_ppo": ("single_pendulum_ppo", "CUDAClassicControlPendulumEnv"),
                 "mountain_car_a2c": ("single_mountain_car", "CUDAClassicControlMountainCarEnv")}
        trainers = {(k, n): rollout_trainer(c, e, n, basedir) for k, (c, e) in pairs.items()
                    for n in (False, True)}
        for tr in trainers.values():
            tr.engine.rollout()
        torch.cuda.synchronize()
        roll = {f"{k} {'norm' if n else 'plain'}": [] for (k, n) in trainers}
        for _ in range(args.rounds):
            for (k, n), tr in trainers.items():
                ms = timed(tr.engine.rollout, 5)
                roll[f"{k} {'norm' if n else 'plain'}"].append(ms / tr.engine.T)
        out["rollout_ms_per_timestep"] = {k: summary(v) for k, v in roll.items()}
        out["rollout_shapes"] = {f"{k}": {"envs": tr.num_envs, "T": tr.engine.T}
                                 for (k, n), tr in trainers.items() if not n}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
