"""Categorical DQN (C51) timings on one GPU, printed as one JSON line (card name and power limit
read in the same run).  With the fc_dims [64, 64] network and N = 51 atoms of
single_cartpole_c51.yaml:

  update_ms  one whole update (window draw + gradients + clipping + Adam) with the native pass
             against the torch autograd loss on the gathered windows, on a full store of 256
             CartPole envs x 4096 slots (~10^6 transitions), at the run config's
             replay_batch_rows (512) and at B = 50 000 sampled windows; with the launches per
             native update;
  pass_ms    the native pass alone (wdb_c51_update_sampled: tile kernel + reduction) at the same
             sizes;
  rollout    one timestep of 10 000 CartPole envs, the one-launch rollout (the categorical head
             reduced over each env's 8 lanes) against the per-step path (torch forward +
             wdb_sample_epsilon_greedy + step kernels).

Every figure is the median over `--rounds` alternated rounds of CUDA-event-timed loops.

    python scripts/bench_c51.py [--rounds 5]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_dqn import gpu_info, timed  # noqa: E402
from bench_qr_dqn import E, SLOTS, fill, pass_fn, setup  # noqa: E402


def make_trainer(name, E=E, T=4, slots=SLOTS):
    """A TrainerDQN of single_cartpole_c51.yaml on E CartPole envs with a store of `slots`
    slots per env."""
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent.cartpole import CUDAClassicControlCartPoleEnv
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_dqn import TrainerDQN

    cfg = load_run_config("single_cartpole_c51")
    cfg["trainer"].update(num_envs=E, train_batch_size=E * T, seed=3, num_episodes=E * 8,
                          replay_slots_per_env=slots, updates_per_iteration=1,
                          replay_warmup_slots=min(64, slots - 8), evaluator=False)
    cfg["saving"].update(basedir=tempfile.mkdtemp(), metrics_log_freq=10 ** 9,
                         model_params_save_freq=10 ** 9)
    env = CUDAClassicControlCartPoleEnv(**cfg["env"])
    w = EnvWrapper(env, num_envs=E, env_backend="numba")
    return TrainerDQN(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                      results_dir=name, verbose=False), cfg


def bench_update(rounds):
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.fused_dqn import FusedC51Update

    tr, cfg = make_trainer("u")
    fill(tr)
    algo = tr.trainers["shared"]
    out = {}
    for B in (int(cfg["trainer"]["replay_batch_rows"]), 50000):
        setup(tr, FusedC51Update, B)
        t = {k: [] for k in ("pass", "update_native", "update_torch")}
        for _ in range(rounds):
            t["pass"].append(timed(pass_fn(tr), 20))
            algo.use_fused_update = True
            t["update_native"].append(timed(lambda: tr._one_update(False, {}), 20))
            algo.use_fused_update = False
            t["update_torch"].append(timed(lambda: tr._one_update(False, {}), 5))
        algo.use_fused_update = True
        n0 = wlib.launch_count()
        tr._one_update(False, {})
        torch.cuda.synchronize()
        launches = wlib.launch_count() - n0
        m = {k: statistics.median(v) for k, v in t.items()}
        out[f"B{B}"] = {"pass_ms": m["pass"],
                        "update_ms": {"native": m["update_native"], "torch": m["update_torch"]},
                        "native_over_torch_speedup": m["update_torch"] / m["update_native"],
                        "launches_per_native_update": launches}
    return out


def bench_rollout(rounds):
    n_envs = 10000
    tr, _ = make_trainer("r", E=n_envs, T=8, slots=16)
    eng = tr.engine
    sa = eng.sa
    assert sa is not None and sa.categorical
    times = {"one_launch": [], "per_step": []}
    for _ in range(rounds):
        for kind in times:
            eng.sa = sa if kind == "one_launch" else None
            times[kind].append(timed(lambda: eng.rollout(epsilon=0.1), 5) / eng.T)
    eng.sa = sa
    return {k: {"ms_per_timestep": statistics.median(v)} for k, v in times.items()} | {
        "envs": n_envs, "speedup": statistics.median(times["per_step"])
        / statistics.median(times["one_launch"])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    print(json.dumps({"gpu": gpu_info(), "rounds": args.rounds, "envs": E, "slots": SLOTS,
                      "fc_dims": [64, 64], "num_atoms": 51, "update": bench_update(args.rounds),
                      "rollout": bench_rollout(args.rounds)}))


if __name__ == "__main__":
    main()
