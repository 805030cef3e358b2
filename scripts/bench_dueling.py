"""Dueling Q network timings on one GPU, printed as one JSON line (card name and power limit read
in the same run).  For the dueling DQN and the dueling C51 head of single_cartpole_dueling_dqn.yaml
and single_cartpole_dueling_c51.yaml (trunk [64], streams [32]: the folded network is [64, 64]),
on a full store of 256 CartPole envs x 4096 slots, at B = 512 (the run configs') and 50 000
sampled windows:

  dueling_ms  the native dueling update's gradient: fold + pass + unfold (4 launches), and fold
              and unfold alone;
  plain_ms    the plain pass at the folded shape (fully_connected_q / fully_connected_categorical_q
              with fc_dims [64, 64]), the lower bound the fold and unfold add to;
  update_ms   one whole update (window draw + gradients + clipping + Adam), native against the
              torch autograd loss on the DuelingHead;
  rollout     one timestep of 10 000 CartPole envs, the one-launch rollout (one fold launch, then
              the folded network) against the per-step path.

Every figure is the median over `--rounds` alternated rounds of CUDA-event-timed loops.

    python scripts/bench_dueling.py [--rounds 5]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_dqn import gpu_info, timed  # noqa: E402
from bench_qr_dqn import E, SLOTS, fill, pass_fn, setup  # noqa: E402

CONFIGS = {"dqn": "single_cartpole_dueling_dqn", "c51": "single_cartpole_dueling_c51"}


def make_trainer(config, name, E=E, T=4, slots=SLOTS, plain=False):
    """A TrainerDQN of `config` on E CartPole envs with a store of `slots` slots per env, without
    prioritized replay; plain: the network of the folded shape (fc_dims [64, 64], no dueling)."""
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent.cartpole import CUDAClassicControlCartPoleEnv
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_dqn import TrainerDQN

    cfg = load_run_config(config)
    for key in ("prioritized_replay", "priority_alpha", "priority_beta", "priority_epsilon"):
        cfg["trainer"].pop(key, None)
    cfg["trainer"].update(num_envs=E, train_batch_size=E * T, seed=3, num_episodes=E * 8,
                          replay_slots_per_env=slots, updates_per_iteration=1,
                          replay_warmup_slots=min(64, slots - 8), evaluator=False)
    if plain:
        model = cfg["policy"]["shared"]["model"]
        for key in ("dueling", "stream_fc_dims"):
            model.pop(key)
        model["fc_dims"] = [64, 64]
    cfg["saving"].update(basedir=tempfile.mkdtemp(), metrics_log_freq=10 ** 9,
                         model_params_save_freq=10 ** 9)
    env = CUDAClassicControlCartPoleEnv(**cfg["env"])
    w = EnvWrapper(env, num_envs=E, env_backend="numba")
    return TrainerDQN(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                      results_dir=name, verbose=False)


def bench_update(kind, rounds):
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.fused_dqn import (
        FusedC51Update, FusedDQNUpdate, FusedDuelingUpdate, fold)

    tr = make_trainer(CONFIGS[kind], f"d{kind}")
    ref = make_trainer(CONFIGS[kind], f"p{kind}", plain=True)
    for t in (tr, ref):
        fill(t)
    algo = tr.trainers["shared"]
    L = wlib.load()
    out = {}
    for B in (512, 50000):
        setup(tr, FusedDuelingUpdate, B)
        setup(ref, FusedC51Update if kind == "c51" else FusedDQNUpdate, B)
        f = tr.fused_updates["shared"]
        unfold = lambda: L.wdb_dueling_unfold_grads(  # noqa: E731
            wlib.stream_ptr(), ctypes.byref(f.online.struct()))
        t = {k: [] for k in ("dueling", "fold", "unfold", "plain", "update_native",
                             "update_torch")}
        for _ in range(rounds):
            t["dueling"].append(timed(pass_fn(tr), 20))
            t["plain"].append(timed(pass_fn(ref), 20))
            t["fold"].append(timed(lambda: fold(f.online, f.target), 50))
            t["unfold"].append(timed(unfold, 50))
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
        out[f"B{B}"] = {"dueling_ms": {"fold_pass_unfold": m["dueling"], "fold": m["fold"],
                                       "unfold": m["unfold"]},
                        "plain_ms": m["plain"],
                        "dueling_over_plain": m["dueling"] / m["plain"],
                        "update_ms": {"native": m["update_native"], "torch": m["update_torch"]},
                        "native_over_torch_speedup": m["update_torch"] / m["update_native"],
                        "launches_per_native_update": launches}
    return out


def bench_rollout(kind, rounds):
    n_envs = 10000
    tr = make_trainer(CONFIGS[kind], f"r{kind}", E=n_envs, T=8, slots=16)
    eng = tr.engine
    sa = eng.sa
    assert sa is not None and sa._dueling is not None
    times = {"one_launch": [], "per_step": []}
    for _ in range(rounds):
        for k in times:
            eng.sa = sa if k == "one_launch" else None
            times[k].append(timed(lambda: eng.rollout(epsilon=0.1), 5) / eng.T)
    eng.sa = sa
    return {k: {"ms_per_timestep": statistics.median(v)} for k, v in times.items()} | {
        "envs": n_envs, "speedup": statistics.median(times["per_step"])
        / statistics.median(times["one_launch"])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    print(json.dumps({"gpu": gpu_info(), "rounds": args.rounds, "envs": E, "slots": SLOTS,
                      "fc_dims": [64], "stream_fc_dims": [32], "num_atoms": 51,
                      **{kind: {"update": bench_update(kind, args.rounds),
                                "rollout": bench_rollout(kind, args.rounds)}
                         for kind in CONFIGS}}))


if __name__ == "__main__":
    main()
