"""Quantile-regression DQN timings on one GPU, printed as one JSON line (card name and power
limit read in the same run).  On a full store of 256 CartPole envs x 4096 slots (~10^6
transitions), with the fc_dims [64, 64] network of the run configs, for B = 256, 4096 and
50 000 sampled windows and N = 8 and 32 quantiles:

  pass_ms    the native pass alone (wdb_qr_dqn_update_sampled: tile kernel + reduction) against
             DQN's (wdb_dqn_update_sampled) on the same windows;
  update_ms  one whole update (window draw + gradients + clipping + Adam) with the native pass,
             with the torch autograd loss on the gathered windows, and DQN's native update;
  launches   per native QR-DQN update.

Every figure is the median over `--rounds` alternated rounds of CUDA-event-timed loops.

    python scripts/bench_qr_dqn.py [--rounds 5]
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

E, SLOTS = 256, 4096


def make_trainer(name, model=None):
    """A TrainerDQN on 256 CartPole envs with a store of 4096 slots per env; `model` replaces
    single_cartpole_dqn.yaml's."""
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent.cartpole import CUDAClassicControlCartPoleEnv
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_dqn import TrainerDQN

    cfg = load_run_config("single_cartpole_dqn")
    cfg["trainer"].update(num_envs=E, train_batch_size=E * 4, seed=3, num_episodes=E * 8,
                          replay_slots_per_env=SLOTS, replay_batch_rows=256,
                          updates_per_iteration=1, replay_warmup_slots=64, evaluator=False)
    if model is not None:
        cfg["policy"]["shared"]["model"] = model
    cfg["saving"].update(basedir=tempfile.mkdtemp(), metrics_log_freq=10 ** 9,
                         model_params_save_freq=10 ** 9)
    env = CUDAClassicControlCartPoleEnv(**cfg["env"])
    w = EnvWrapper(env, num_envs=E, env_backend="numba")
    return TrainerDQN(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                      results_dir=name, verbose=False)


def fill(tr):
    """A full store of random transitions (the same for every trainer)."""
    eng = tr.engine
    g = torch.Generator(device="cuda").manual_seed(0)
    with torch.no_grad():
        eng._tensor("processed_observations_batch_shared").normal_(generator=g)
        eng._tensor("sampled_actions_batch_shared").random_(0, 2, generator=g)
        eng._tensor("rewards_batch_shared").fill_(1.0)
        eng._tensor("done_flags_batch").copy_(
            (torch.rand(eng._tensor("done_flags_batch").shape, device="cuda", generator=g)
             < 0.01).to(torch.int32))
    eng.ring_filled, eng.ring_cursor = SLOTS, 0


def setup(tr, fused_cls, B):
    algo, q, t = tr.trainers["shared"], tr.q_models["shared"], tr.target_q_models["shared"]
    tr.replay_windows["shared"] = torch.zeros((B, 2), dtype=torch.int32, device="cuda")
    tr.fused_updates["shared"] = fused_cls(algo, q, t, E, 1, SLOTS, B)
    tr._sample_replay_windows("shared")
    for p in q.parameters():
        if p.grad is None:
            p.grad = torch.zeros_like(p)


def pass_fn(tr):
    eng, f = tr.engine, tr.fused_updates["shared"]
    args = (eng._tensor("processed_observations_batch_shared"),
            eng._tensor("sampled_actions_batch_shared"), eng._tensor("rewards_batch_shared"),
            eng._tensor("done_flags_batch"), tr.replay_windows["shared"])
    return lambda: f.launch(*args)


def main():
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.fused_dqn import FusedDQNUpdate, FusedQRDQNUpdate

    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    dqn = make_trainer("dqn")
    qr = {N: make_trainer(f"qr{N}", model={
        "type": "fully_connected_quantile_q", "fc_dims": [64, 64], "num_quantiles": N,
        "model_ckpt_filepath": ""}) for N in (8, 32)}
    for tr in [dqn, *qr.values()]:
        fill(tr)
    out = {}
    for B in (256, 4096, 50000):
        setup(dqn, FusedDQNUpdate, B)
        for N, tr in qr.items():
            setup(tr, FusedQRDQNUpdate, B)
            algo = tr.trainers["shared"]
            t = {k: [] for k in ("pass_qr", "pass_dqn", "update_qr", "update_torch",
                                 "update_dqn")}
            for _ in range(args.rounds):
                t["pass_qr"].append(timed(pass_fn(tr), 20))
                t["pass_dqn"].append(timed(pass_fn(dqn), 20))
                algo.use_fused_update = True
                t["update_qr"].append(timed(lambda: tr._one_update(False, {}), 20))
                algo.use_fused_update = False
                t["update_torch"].append(timed(lambda: tr._one_update(False, {}), 20))
                t["update_dqn"].append(timed(lambda: dqn._one_update(False, {}), 20))
            algo.use_fused_update = True
            n0 = wlib.launch_count()
            tr._one_update(False, {})
            torch.cuda.synchronize()
            launches = wlib.launch_count() - n0
            m = {k: statistics.median(v) for k, v in t.items()}
            out[f"B{B}_N{N}"] = {
                "pass_ms": {"qr_dqn": m["pass_qr"], "dqn": m["pass_dqn"]},
                "update_ms": {"qr_dqn_native": m["update_qr"], "qr_dqn_torch": m["update_torch"],
                              "dqn_native": m["update_dqn"]},
                "native_over_torch_speedup": m["update_torch"] / m["update_qr"],
                "launches_per_native_update": launches}
    print(json.dumps({"gpu": gpu_info(), "rounds": args.rounds, "envs": E, "slots": SLOTS,
                      "fc_dims": [64, 64], "results": out}))


if __name__ == "__main__":
    main()
