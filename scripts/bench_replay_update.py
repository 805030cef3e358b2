"""Replay-buffer update passes on the GPU (E = 10 000 Pendulum envs, ring filled to capacity):
each sampled pass (wdb_*_update_sampled) against its torch path on the gathered batch, in
alternated rounds of one process; the sampled DDPG pass against the ring pass at equal row
count (the cost of scattered rows); the window draw; and whole iterations of TrainerDDPG/TD3/SAC
at updates_per_iteration 1 and 4 with the launches per update.

    python scripts/bench_replay_update.py [--rounds 7] [--out replay.json]

Times are CUDA events around `--reps` back-to-back calls; the card's name and power limit are
read in the same run.  Fails without a GPU."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    return q


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps * 1e3            # microseconds per call


def stats(xs):
    return {"median_us": round(statistics.median(xs), 1), "min_us": round(min(xs), 1),
            "max_us": round(max(xs), 1)}


def trainer(algo, E, T, basedir, **replay):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent import classic_control as cc
    from warp_drive_b200.training import trainer_ddpg, trainer_sac, trainer_td3
    from warp_drive_b200.training.trainer import load_run_config

    cfg = load_run_config({"DDPG": "single_pendulum", "TD3": "single_pendulum_td3",
                           "SAC": "single_pendulum_sac"}[algo])
    cfg["trainer"].update(num_envs=E, train_batch_size=E * T, num_episodes=E * 100, seed=1)
    cfg["trainer"].update(replay)
    cfg["trainer"]["evaluator"] = False
    cfg["env"].update(reset_pool_size=min(E, 10000))
    cfg["saving"].update(basedir=basedir, metrics_log_freq=10 ** 9, model_params_save_freq=10 ** 9)
    env = cc.CUDAClassicControlPendulumEnv(**cfg["env"])
    w = EnvWrapper(env, num_envs=E, env_backend="numba")
    cls = {"DDPG": trainer_ddpg.TrainerDDPG, "TD3": trainer_td3.TrainerTD3,
           "SAC": trainer_sac.TrainerSAC}[algo]
    return cls(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
               results_dir="bench", verbose=False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--envs", type=int, default=10000)
    ap.add_argument("--slots", type=int, default=105)     # ~10^6 transitions at 10 000 envs
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_replay_update.py needs a GPU")
    from warp_drive_b200 import lib as wlib

    E, T = args.envs, 5
    result = {"card": card(), "envs": E, "slots_per_env": args.slots, "passes": {},
              "iterations": {}}
    tmp = tempfile.mkdtemp()
    for algo in ("DDPG", "TD3", "SAC"):
        for B in (256, 4096, 50000):
            tr = trainer(algo, E, T, tmp, replay_slots_per_env=args.slots, replay_batch_rows=B)
            while not tr.engine.isfull():
                tr._generate_rollout_batch()
            a = tr.trainers["shared"]
            tr._sample_replay_windows("shared")

            def critic(fused):
                a.use_fused_update = fused
                if algo == "DDPG":
                    f = tr.fused_updates["shared"]
                    return (tr._fused_gradients("shared", f, False) if fused
                            else tr._torch_replay_gradients("shared", False))
                return tr._critic_gradients("shared", False)

            passes = {"critic" if algo != "DDPG" else "update": critic}
            if algo != "DDPG":
                def actor(fused):
                    a.use_fused_update = fused
                    return tr._actor_gradients("shared", False)
                passes["actor"] = actor
            for name, fn in passes.items():
                times = {True: [], False: []}
                for fused in (True, False):              # warm-up of both paths
                    timed(lambda: fn(fused), 3)
                for _ in range(args.rounds):
                    for fused in (True, False):
                        times[fused].append(timed(lambda: fn(fused), args.reps))
                row = {"sampled_kernels": stats(times[True]), "torch_gather": stats(times[False])}
                row["speedup_of_medians"] = round(
                    row["torch_gather"]["median_us"] / row["sampled_kernels"]["median_us"], 2)
                result["passes"][f"{algo} {name} B={B}"] = row
            a.use_fused_update = True
            if B == 256:
                draw = [timed(lambda: tr._sample_replay_windows("shared"), 200)
                        for _ in range(args.rounds)]
                result.setdefault("window_draw", {})[f"{algo} B={B}"] = stats(draw)
            del tr
            torch.cuda.empty_cache()

    # scattered rows against streamed rows: the ring pass over every window of a T + n_step - 1
    # ring (45 000 rows + the last window's 5 000) and the sampled pass over as many rows of
    # the long ring
    ring = trainer("DDPG", E, T, tmp)
    while not ring.engine.isfull():
        ring._generate_rollout_batch()
    rows = ring.fused_updates["shared"].rows
    long = trainer("DDPG", E, T, tmp, replay_slots_per_env=args.slots, replay_batch_rows=rows)
    while not long.engine.isfull():
        long._generate_rollout_batch()
    long._sample_replay_windows("shared")
    fns = {"ring_pass": lambda: ring._fused_gradients("shared", ring.fused_updates["shared"],
                                                      False),
           "sampled_pass": lambda: long._fused_gradients("shared", long.fused_updates["shared"],
                                                         False)}
    times = {k: [] for k in fns}
    for k, fn in fns.items():
        timed(fn, 3)
    for _ in range(args.rounds):
        for k, fn in fns.items():
            times[k].append(timed(fn, args.reps))
    result["ddpg_equal_rows"] = {"rows": rows, **{k: stats(v) for k, v in times.items()}}
    del ring, long
    torch.cuda.empty_cache()

    # whole iterations (rollout + updates) of the replay run configs' sizes
    for algo in ("DDPG", "TD3", "SAC"):
        for updates in (1, 4):
            tr = trainer(algo, 256, 4, tmp, replay_slots_per_env=4096, replay_batch_rows=1024,
                         updates_per_iteration=updates, replay_warmup_slots=16)
            for it in range(8):
                tr._generate_rollout_batch()
                tr._update_model_params(1)

            def iteration():
                tr._generate_rollout_batch()
                tr._update_model_params(1)

            n0 = wlib.launch_count()
            tr._update_model_params(1)
            launches = (wlib.launch_count() - n0) / updates
            xs = [timed(iteration, 50) for _ in range(args.rounds)]
            result["iterations"][f"{algo} updates_per_iteration={updates}"] = {
                **stats(xs), "native_launches_per_update": launches}
            del tr
            torch.cuda.empty_cache()
    line = json.dumps(result, indent=1)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line)


if __name__ == "__main__":
    main()
