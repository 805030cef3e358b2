"""Prioritized-replay timings on one GPU, printed as one JSON line (card name and power limit read
in the same run):

  store     per call, over stores of ~10^6 and ~10^7 windows (256 agent rows x C slots):
            wdb_per_sample_windows at B = 256, 4096 and 50 000 (descent + weights),
            wdb_per_set_priorities at the same B (leaf writes + tree repair), and wdb_per_admit
            of one single_cartpole_dqn.yaml rollout (4 slots x 256 rows); with launches per call;
  update    one whole TrainerDQN update at single_cartpole_dqn.yaml sizes (256 envs x 4096
            slots, B = 512): uniform (wdb_replay_sample_windows + wdb_dqn_update_sampled) against
            prioritized (wdb_per_sample_windows + wdb_dqn_update_prioritized +
            wdb_per_set_priorities), both followed by clipping + Adam; with launches per update.

Every figure is the median over `--rounds` alternated rounds of CUDA-event-timed loops of
back-to-back calls.

    python scripts/bench_per.py [--rounds 5]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_dqn import gpu_info, timed  # noqa: E402

ROWS = 256


def filled_store(C, B_max):
    """A full store of C slots x 256 rows with varied priorities and a fresh tree."""
    from warp_drive_b200.training.utils.prioritized_replay import PrioritizedReplay

    n_step = 3
    st = PrioritizedReplay(C, ROWS, n_step, B_max, 0.6, 1e-6, "cuda")
    st.admit((0, 0), (C - n_step, C - n_step))
    st.admit((C - n_step, C - n_step), (0, C))
    g = torch.Generator(device="cuda").manual_seed(0)
    for _ in range(40):
        w = torch.stack([torch.randint(0, C, (B_max,), device="cuda", generator=g),
                         torch.randint(0, ROWS, (B_max,), device="cuda", generator=g)],
                        dim=1).to(torch.int32).contiguous()
        q = torch.randn(B_max, device="cuda", generator=g) * 3
        st.set_priorities(w, q, torch.zeros_like(q), 0, C)
    return st


def bench_store(rounds):
    from warp_drive_b200 import lib as wlib

    out = {}
    for C in (3907, 39063):                            # ~10^6 and ~10^7 windows
        st = filled_store(C, 50000)
        st.set_beta(0.5)
        res = {"windows": C * ROWS, "levels": st.levels}
        g = torch.Generator(device="cuda").manual_seed(1)
        ops = {}
        cursor = [0]                                   # the ring is full: oldest = cursor
        for B in (256, 4096, 50000):
            win = torch.zeros((B, 2), dtype=torch.int32, device="cuda")
            counter = [0]

            def sample(win=win, counter=counter):
                counter[0] += 1
                st.sample(win, 9, counter[0])

            sample()
            q = torch.randn(B, device="cuda", generator=g)
            r = torch.zeros_like(q)
            ops[f"sample_B{B}"] = sample
            ops[f"set_priorities_B{B}"] = (
                lambda win=win, q=q, r=r: st.set_priorities(win, q, r, cursor[0], C))

        def admit():                                   # one rollout of 4 slots
            before = (cursor[0], C)
            cursor[0] = (cursor[0] + 4) % C
            st.admit(before, (cursor[0], C))

        ops["admit_T4"] = admit
        times = {k: [] for k in ops}
        for _ in range(rounds):
            for k, fn in ops.items():
                times[k].append(timed(fn, 50))
        for k, fn in ops.items():
            n0 = wlib.launch_count()
            fn()
            res[k] = {"ms": statistics.median(times[k]), "launches": wlib.launch_count() - n0}
        out[f"C{C}"] = res
    return out


def make_trainer(prioritized, name):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent.cartpole import CUDAClassicControlCartPoleEnv
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_dqn import TrainerDQN

    cfg = load_run_config("single_cartpole_dqn_prioritized" if prioritized
                          else "single_cartpole_dqn")
    cfg["trainer"].update(seed=3, evaluator=False)
    cfg["saving"].update(basedir=tempfile.mkdtemp(), metrics_log_freq=10 ** 9,
                         model_params_save_freq=10 ** 9)
    env = CUDAClassicControlCartPoleEnv(**cfg["env"])
    w = EnvWrapper(env, num_envs=cfg["trainer"]["num_envs"], env_backend="numba")
    return TrainerDQN(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                      results_dir=name, verbose=False)


def bench_update(rounds):
    from warp_drive_b200 import lib as wlib

    trs = {"uniform": make_trainer(False, "u"), "prioritized": make_trainer(True, "p")}
    for tr in trs.values():
        # fill the whole store with rollouts (the admits build the priorities as in training)
        while tr.engine.ring_filled < tr.ring_capacity:
            tr._generate_rollout_batch()
    times = {k: [] for k in trs}
    for _ in range(rounds):
        for k, tr in trs.items():
            times[k].append(timed(lambda tr=tr: tr._one_update(False, {}), 50))
    out = {}
    for k, tr in trs.items():
        n0 = wlib.launch_count()
        tr._one_update(False, {})
        out[k] = {"ms": statistics.median(times[k]), "launches": wlib.launch_count() - n0}
    t = trs["uniform"]
    out.update(rows=t.fused_updates["shared"].rows, envs=t.num_envs, slots=t.ring_capacity,
               ratio=out["prioritized"]["ms"] / out["uniform"]["ms"])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    res = {"gpu": gpu_info(), "rounds": args.rounds, "store": bench_store(args.rounds),
           "update": bench_update(args.rounds)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
