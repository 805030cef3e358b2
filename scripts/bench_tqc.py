"""TQC timings on one GPU, printed as one JSON line (card name and power limit read in the same
run):

  passes    the critic pass and the actor pass each, native (wdb_tqc_*_update_sampled, two
            launches each) against the torch path (gather + autograd of the same loss), at the
            run shape of single_pendulum_tqc_replay.yaml: a full store of 256 Pendulum envs x
            4096 slots, [64, 64] networks, two critics of 25 quantiles, 2 dropped per critic,
            B = 1024 sampled windows;
  update    one whole update of that shape (window draw, noise draws, both passes, clipping +
            Adam of the critics and the actor, Adam of log_alpha, target tracking), native and
            torch, with the launches of a native update.

Every figure is the median over `--rounds` alternated rounds of CUDA-event-timed loops.

    python scripts/bench_tqc.py [--rounds 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else torch.cuda.get_device_name()


def make_trainer():
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent.classic_control import CUDAClassicControlPendulumEnv
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_tqc import TrainerTQC

    cfg = load_run_config("single_pendulum_tqc_replay")
    cfg["trainer"].update(seed=3, updates_per_iteration=1)
    cfg["trainer"]["evaluator"] = False
    cfg["saving"].update(basedir=tempfile.mkdtemp(), metrics_log_freq=10 ** 9,
                         model_params_save_freq=10 ** 9)
    env = CUDAClassicControlPendulumEnv(**cfg["env"])
    w = EnvWrapper(env, num_envs=cfg["trainer"]["num_envs"], env_backend="numba")
    return TrainerTQC(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                      results_dir="b", verbose=False)


def timed(fn, n):
    """ms per call of fn over n calls (CUDA events, after one warm call)."""
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def main():
    from warp_drive_b200 import lib as wlib

    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    tr = make_trainer()
    eng = tr.engine
    g = torch.Generator(device="cuda").manual_seed(0)
    with torch.no_grad():                          # a full store of random transitions
        eng._tensor("processed_observations_batch_shared").normal_(generator=g)
        eng._tensor("sampled_actions_batch_shared").uniform_(-2.0, 2.0, generator=g)
        eng._tensor("rewards_batch_shared").uniform_(-16.0, 0.0, generator=g)
        done = eng._tensor("done_flags_batch")
        done.copy_((torch.rand(done.shape, device="cuda", generator=g) < 0.01).to(torch.int32))
    eng.ring_filled, eng.ring_cursor = eng.ring_capacity, 0
    algo = tr.trainers["shared"]
    assert "shared" in tr.fused_updates
    tr._sample_replay_windows("shared")
    tr.critic_noise["shared"].normal_(generator=g)
    tr.actor_noise["shared"].normal_(generator=g)
    work = {"critic": lambda: tr._critic_gradients("shared", False),
            "actor": lambda: tr._actor_gradients("shared", False),
            "update": lambda: tr._one_update(False, {})}
    times = {(k, f): [] for k in work for f in (True, False)}
    for _ in range(args.rounds):
        for k, fn in work.items():
            for fused in (True, False):
                algo.use_fused_update = fused
                times[(k, fused)].append(timed(fn, 50))
    algo.use_fused_update = True
    n0 = wlib.launch_count()
    tr._one_update(False, {})
    torch.cuda.synchronize()
    launches = wlib.launch_count() - n0
    res = {"gpu": gpu_info(), "rounds": args.rounds, "envs": tr.num_envs,
           "slots_per_env": tr.ring_capacity, "rows": tr.fused_updates["shared"].rows,
           "launches_per_native_update": launches}
    for k in work:
        f, t = statistics.median(times[(k, True)]), statistics.median(times[(k, False)])
        res[k] = {"native_ms": f, "torch_ms": t, "speedup": t / f}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
