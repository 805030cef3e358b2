"""Noisy Q network timings on one GPU, printed as one JSON line (card name and power limit read in
the same run).  For the noisy DQN of single_cartpole_noisy_dqn.yaml (fc_dims [64, 64], a noisy
output layer) and the noisy dueling C51 of single_cartpole_rainbow.yaml (trunk [64], noisy
streams [32]), on a full store of 256 CartPole envs x 4096 slots, at B = 512 (the run configs')
and 50 000 sampled windows:

  noisy_ms    the native noisy update's gradient: materialize + [fold +] pass + [unfold +] grads,
              and materialize and grads alone (per call, host work included);
  kernel_ms   the materialize and grads kernels' own device time (torch.profiler);
  plain_ms    the same network without noise (noisy: false) through its native update's gradient
              (the plain DQN pass, or fold + C51 pass + unfold), the lower bound the noise adds to;
  update_ms   one whole update (window draw + gradients + clipping + Adam), native against the
              torch autograd loss on the noisy head;
  rollout     one timestep of 10 000 CartPole envs: noisy DQN on the one-launch rollout's noisy
              kind and on the per-step path (one noise draw per step), against the same network
              without noise on the Q kind and on the per-step path (Rainbow: per step only);
  iteration   one training iteration of the run config (256 envs, a 4-step rollout, 2 updates;
              prioritized replay for Rainbow), noisy against the config without noise.

Every figure is the median over `--rounds` alternated rounds of CUDA-event-timed loops.

    python scripts/bench_noisy.py [--rounds 5]
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

CONFIGS = {"dqn": "single_cartpole_noisy_dqn", "rainbow": "single_cartpole_rainbow"}


def make_trainer(config, name, E=E, T=4, slots=SLOTS, noisy=True, per=False):
    """A TrainerDQN of `config` on E CartPole envs with a store of `slots` slots per env, without
    prioritized replay unless `per`; noisy=False: the same network without noise."""
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent.cartpole import CUDAClassicControlCartPoleEnv
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_dqn import TrainerDQN

    cfg = load_run_config(config)
    if not per:
        for key in ("prioritized_replay", "priority_alpha", "priority_beta", "priority_epsilon"):
            cfg["trainer"].pop(key, None)
    cfg["trainer"].update(num_envs=E, train_batch_size=E * T, seed=3, num_episodes=E * 8,
                          replay_slots_per_env=slots, replay_warmup_slots=min(64, slots - 8),
                          evaluator=False)
    if not per:
        cfg["trainer"]["updates_per_iteration"] = 1
    if not noisy:
        model = cfg["policy"]["shared"]["model"]
        for key in ("noisy", "noisy_sigma0"):
            model.pop(key, None)
    cfg["saving"].update(basedir=tempfile.mkdtemp(), metrics_log_freq=10 ** 9,
                         model_params_save_freq=10 ** 9)
    env = CUDAClassicControlCartPoleEnv(**cfg["env"])
    w = EnvWrapper(env, num_envs=E, env_backend="numba")
    return TrainerDQN(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                      results_dir=name, verbose=False)


def bench_update(kind, rounds):
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.fused_dqn import (
        FusedDQNUpdate, FusedDuelingUpdate, FusedNoisyUpdate, materialize, noisy_grads)

    tr = make_trainer(CONFIGS[kind], f"n{kind}")
    ref = make_trainer(CONFIGS[kind], f"p{kind}", noisy=False)
    for t in (tr, ref):
        fill(t)
    algo = tr.trainers["shared"]
    out = {}
    for B in (512, 50000):
        setup(tr, lambda *a: FusedNoisyUpdate(*a, tr.seed), B)
        setup(ref, FusedDuelingUpdate if kind == "rainbow" else FusedDQNUpdate, B)
        f = tr.fused_updates["shared"]
        t = {k: [] for k in ("noisy", "materialize", "grads", "plain", "update_native",
                             "update_torch")}
        for _ in range(rounds):
            t["noisy"].append(timed(pass_fn(tr), 20))
            t["plain"].append(timed(pass_fn(ref), 20))
            t["materialize"].append(timed(lambda: materialize(f.online, f.target, tr.seed, 1),
                                          50))
            t["grads"].append(timed(lambda: noisy_grads(f.online), 50))
            algo.use_fused_update = True
            t["update_native"].append(timed(lambda: tr._one_update(False, {}), 20))
            algo.use_fused_update = False
            t["update_torch"].append(timed(lambda: tr._one_update(False, {}), 5))
        algo.use_fused_update = True
        kernel = kernel_ms(lambda: (materialize(f.online, f.target, tr.seed, 1),
                                    noisy_grads(f.online)), 50)
        n0 = wlib.launch_count()
        tr._one_update(False, {})
        torch.cuda.synchronize()
        launches = wlib.launch_count() - n0
        m = {k: statistics.median(v) for k, v in t.items()}
        out[f"B{B}"] = {"noisy_ms": {"gradient": m["noisy"], "materialize": m["materialize"],
                                     "grads": m["grads"]},
                        "kernel_ms": kernel,
                        "plain_ms": m["plain"],
                        "noisy_over_plain": m["noisy"] / m["plain"],
                        "update_ms": {"native": m["update_native"], "torch": m["update_torch"]},
                        "native_over_torch_speedup": m["update_torch"] / m["update_native"],
                        "launches_per_native_update": launches}
    return out


def kernel_ms(fn, n):
    """Device time per call of the noisy kernels fn launches (torch.profiler, after a warm call)."""
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for name in ("noisy_materialize_kernel", "noisy_grads_kernel"):
            if name in e.key:
                out[name] = e.device_time_total / 1000.0 / n
    return out


def bench_rollout(kind, rounds):
    n_envs = 10000
    noisy = make_trainer(CONFIGS[kind], f"rn{kind}", E=n_envs, T=8, slots=16)
    plain = make_trainer(CONFIGS[kind], f"rp{kind}", E=n_envs, T=8, slots=16, noisy=False)
    assert plain.engine.sa is not None
    assert (noisy.engine.sa is not None) == (kind == "dqn")
    sas = {"noisy": noisy.engine.sa, "plain": plain.engine.sa}
    cases = [("noisy", "per_step"), ("plain", "per_step"), ("plain", "one_launch")]
    if kind == "dqn":
        cases.append(("noisy", "one_launch"))
    times = {f"{n}_{p}": [] for n, p in cases}
    for _ in range(rounds):
        for n, p in cases:
            tr = noisy if n == "noisy" else plain
            tr.engine.sa = sas[n] if p == "one_launch" else None
            times[f"{n}_{p}"].append(timed(lambda: tr.engine.rollout(epsilon=0.0), 5) / tr.engine.T)
    noisy.engine.sa, plain.engine.sa = sas["noisy"], sas["plain"]
    return {k: {"ms_per_timestep": statistics.median(v)} for k, v in times.items()} | {
        "envs": n_envs}


def bench_iteration(kind, rounds):
    """One iteration of the run config as it trains (prioritized replay for Rainbow)."""
    trs = {n: make_trainer(CONFIGS[kind], f"i{kind}{n}", noisy=n, per=True, T=4)
           for n in (True, False)}
    for tr in trs.values():
        for _ in range(20):                    # past the warm-up slots
            tr._generate_rollout_batch()

    def step(tr):
        tr._generate_rollout_batch()
        tr._update_model_params(1)
    times = {True: [], False: []}
    for _ in range(rounds):
        for n, tr in trs.items():
            times[n].append(timed(lambda: step(tr), 20))
    return {"noisy_ms": statistics.median(times[True]),
            "plain_ms": statistics.median(times[False]),
            "noisy_one_launch_rollout": trs[True].engine.sa is not None,
            "plain_one_launch_rollout": trs[False].engine.sa is not None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    print(json.dumps({"gpu": gpu_info(), "rounds": args.rounds, "envs": E, "slots": SLOTS,
                      **{kind: {"update": bench_update(kind, args.rounds),
                                "rollout": bench_rollout(kind, args.rounds),
                                "iteration": bench_iteration(kind, args.rounds)}
                         for kind in CONFIGS}}))


if __name__ == "__main__":
    main()
